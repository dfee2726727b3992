"""Variant-M packed batching vs sequential calls on one GPU: the 8B synthetic model and the M inputs of bench.py's
measure_variant_m (text_cfg 2.5, image_cfg 4.0, 128 text steps, 64 image steps), N in {1, 2, 4} requests whose prompts differ in
length (T = 32, 49, 15, 43 text tokens after the input image), at 512x512 (1024 MagViT tokens, L = 2341 + T - 32) and 256x256
(256 tokens). For each size and N, one `interleave_generate_batch` call and N sequential `interleave_generate` calls are timed
(CUDA events, alternating in one process after a warm-up of both paths) and their outputs compared. A second part times one
packed forward over the [cond; uncond] sequences of N requests with M's text-step row windows against the same forward without
windows. The executed FLOP are counted from the forward shapes (both paths run the same last-block windows). Prints one JSON line;
the GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_batch_m.py [--reps 1] [--warmup 1] [--sizes 32,16] [--ns 1,2,4] [--fwd-iters 20] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench import CODEBOOK, MASK, MODEL_8B, model_namespace, synthetic_tensors  # noqa: E402
from bench_batch import gpu_info  # noqa: E402

TEXTS = (32, 49, 15, 43)  # prompt text tokens per request; bench.py's M input has 32
TVOC, SOI, EOI, BOS = 126349, 126085, 126086, 126080
GEN = dict(text_cfg=2.5, image_cfg=4.0, text_steps=128, image_steps=64)
MAX_SEQ = 256  # generated text positions


def build(device: str, max_batch: int, seed: int = 1000):
    from mmada_parallel_b200.mmada import MMadaModelLM
    ns = model_namespace(MODEL_8B)
    ns.mask_token_id = MASK
    m = MMadaModelLM(ns, max_seq_len=MODEL_8B["max_sequence_length"], max_batch=max_batch, device=device)
    for name, t in synthetic_tensors(MODEL_8B, device, seed):
        assert m.set_weight(name, t)
    m.load_state_dict({}, strict=True)
    torch.cuda.synchronize()
    return m


def requests(n: int, grid: int, device: str) -> list:
    """measure_variant_m's request (input image ids + a text prompt; the uncond prompt differs in its text), T text tokens each."""
    class Tok:
        bos_token_id = BOS

        def __len__(self):
            return TVOC

    n_vq = grid * grid
    conf = SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=n_vq, codebook_size=CODEBOOK)),
                           dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=MAX_SEQ)))
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(i)
        T = TEXTS[i]
        inp = torch.cat([torch.tensor([126340, SOI]), torch.randint(TVOC, TVOC + CODEBOOK, (n_vq,), generator=g), torch.tensor([EOI]),
                         torch.randint(0, 126000, (T,), generator=g)])
        unc = inp.clone()
        unc[-T:] = torch.randint(0, 126000, (T,), generator=g)
        out.append(dict(input_ids=inp, uncond_input_ids=unc, reserved_token_mapping={"<|soi|>": SOI, "<|eoi|>": EOI}, config=conf,
                        uni_prompting=SimpleNamespace(text_tokenizer=Tok()), generator=torch.Generator(device=device).manual_seed(42 + i),
                        **GEN))
    return out


def forward_flops(lens, windows, rows_a, rows_b) -> float:
    """FLOP of one packed forward over sequences `lens` whose last block runs on `windows` ((lo, hi) or None per sequence), with
    rows_a text rows x V and rows_b image rows x the codebook."""
    c = MODEL_8B
    d, ff, V, nl = c["d_model"], c["mlp_hidden_size"], c["vocab_size"], c["n_layers"]
    M = sum(lens)
    f = (nl - 1) * (2.0 * M * d * (4 * d + 3 * ff) + 4.0 * d * sum(L * L for L in lens))
    for L, w in zip(lens, windows):
        q = L if w is None else w[1] - w[0]
        f += 2.0 * L * d * 3 * d + 2.0 * q * d * (d + 3 * ff) + 4.0 * d * q * L
    return f + 2.0 * d * (rows_a * V + rows_b * CODEBOOK)


def sample_flops(reqs) -> float:
    """Executed FLOP of the requests' loops: per step one forward over [cond; uncond] with interleave_generate's windows."""
    from mmada_parallel_b200.schedule import image_generation_step_indices
    total = 0.0
    for r in reqs:
        n_vq, P = r["config"].model.mmada.num_vq_tokens, r["input_ids"].numel()
        L = P + n_vq + MAX_SEQ + 2
        img = set(image_generation_step_indices(r["text_steps"], r["image_steps"]))
        for s in range(r["text_steps"]):
            w = None if L < 1024 else ((P + 1, L) if s in img else (L - MAX_SEQ, L))
            total += forward_flops([L, L], [w, w], 2 * MAX_SEQ, 2 * n_vq if s in img else 0)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=1, help="timed repetitions of each (size, N) pair")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="32,16", help="VQ grids (32: 512x512, 16: 256x256)")
    ap.add_argument("--ns", default="1,2,4")
    ap.add_argument("--fwd-iters", type=int, default=20, help="timed packed forwards per arm (0: skip the forward part)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch_m: needs a CUDA device (H100)")
    from mmada_parallel_b200.generators.batch import interleave_generate_batch

    device = "cuda:0"
    torch.cuda.set_device(device)
    ns = [int(x) for x in args.ns.split(",")]
    model = build(device, max_batch=2 * max(ns))

    def run(reqs, batched):
        return interleave_generate_batch(model, reqs) if batched else [model.interleave_generate(**r) for r in reqs]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def n_diff(a, b):
        return sum(int((x[0] != y[0]).sum()) + int((x[1] != y[1]).sum()) for x, y in zip(a, b))

    res = {"metric": "variant_m_packed_batch_vs_sequential_tokens_per_s", "model": "8B synthetic (bench.py), bf16",
           "prompt_text_tokens": list(TEXTS), "gen": GEN, "runs": [], "forward": []}
    t_start = time.time()
    with torch.no_grad():
        for grid in (int(x) for x in args.sizes.split(",")):
            for _ in range(args.warmup):
                run(requests(1, grid, device), True)
                run(requests(1, grid, device), False)
            for n in ns:
                tokens = n * (grid * grid + MAX_SEQ)
                ms, outs = {True: [], False: []}, {}
                for rep in range(args.reps):
                    for batched in ((True, False) if rep % 2 == 0 else (False, True)):  # alternating order
                        t, outs[batched] = timed(lambda: run(requests(n, grid, device), batched))
                        ms[batched].append(t)
                reqs = requests(n, grid, device)
                fl = sample_flops(reqs)
                row = {"image": f"{grid * 16}x{grid * 16}", "n": n,
                       "lengths": [r["input_ids"].numel() + grid * grid + MAX_SEQ + 2 for r in reqs], "pflop": round(fl / 1e15, 3)}
                for batched, key in ((True, "batch"), (False, "sequential")):
                    mean = sum(ms[batched]) / len(ms[batched])
                    row[key] = {"ms": [round(v, 1) for v in ms[batched]], "tokens_per_s": round(tokens / (mean / 1e3), 2),
                                "tflops": round(fl / (mean / 1e3) / 1e12, 1)}
                row["ratio_batch_over_sequential"] = round(row["batch"]["tokens_per_s"] / row["sequential"]["tokens_per_s"], 4)
                row["differing_ids_default_options"] = n_diff(outs[True], outs[False])
                row["total_ids"] = sum(x[0].numel() + x[1].numel() for x in outs[False])
                res["runs"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
        # one packed forward over [cond; uncond] of N requests at 512x512 on a text step: M's text windows against none
        if args.fwd_iters:
            for n in ns:
                reqs = requests(n, 32, device)
                seqs, wins = [], []
                for r in reqs:
                    L = r["input_ids"].numel() + 1024 + MAX_SEQ + 2
                    ids = torch.cat([r["input_ids"], torch.full((L - r["input_ids"].numel(),), MASK)]).to(device)
                    seqs += [ids, ids]
                    wins += [(L - MAX_SEQ, L)] * 2
                lens = [s.numel() for s in seqs]
                offs = [sum(lens[:j]) for j in range(len(lens))]
                rows = torch.cat([torch.arange(o + L - MAX_SEQ, o + L, dtype=torch.int32) for o, L in zip(offs, lens)]).to(device)
                ids = torch.cat(seqs)
                out = torch.empty((rows.numel(), model.vocab_rows), dtype=torch.bfloat16, device=device)

                def fwd(w):
                    for _ in range(args.fwd_iters):
                        model.forward_rows_packed(ids, lens, rows_a=rows, out_a=out, row_windows=w)

                for w in (wins, None):
                    fwd(w)  # warm-up
                ms = {"windows": [], "none": []}
                for rep in range(4):
                    for key in (("windows", "none") if rep % 2 == 0 else ("none", "windows")):
                        ms[key].append(timed(lambda: fwd(wins if key == "windows" else None))[0] / args.fwd_iters)
                row = {"n_requests": n, "sequences": len(lens), "lengths": lens}
                for key, w in (("windows", wins), ("none", [None] * len(lens))):
                    fl = forward_flops(lens, w, rows.numel(), 0)
                    mean = sum(ms[key]) / len(ms[key])
                    row[key] = {"ms": round(mean, 3), "ms_reps": [round(v, 3) for v in ms[key]], "tflop": round(fl / 1e12, 2),
                                "tflops": round(fl / (mean / 1e3) / 1e12, 1)}
                row["time_saved_pct"] = round(100.0 * (1 - row["windows"]["ms"] / row["none"]["ms"]), 2)
                row["flop_saved_pct"] = round(100.0 * (1 - row["windows"]["tflop"] / row["none"]["tflop"]), 2)
                res["forward"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    res["gpu"] = gpu_info()
    res["wall_s"] = round(time.time() - t_start, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
