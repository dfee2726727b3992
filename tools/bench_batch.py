"""Packed batching vs sequential calls on one GPU: the 8B synthetic model and inputs of bench.py, N in {1, 2, 4} requests with
distinct prompt lengths (P = 40, 57, 23, 51), at 512x512@64 (grid 32) and 256x256@64 (grid 16). For each size and N, one
`generate_ti2ti_batch` call and N sequential `generate_ti2ti` calls are timed (CUDA events, alternating in one process after a
warm-up of both paths), and their ids compared (number of differing ids with default options). One extra check runs the
batch and the sequential calls with GEMM split-K and the attention split tail off and compares the ids bit for bit.
The executed FLOP are counted from the forward shapes of each path (the sequential path's last block runs on its row window).
Prints one JSON line; the GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_batch.py [--reps 1] [--warmup 1] [--sizes 32,16] [--ns 1,2,4] [--exact-grid 16] [--out FILE]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import CODEBOOK, GEN, MODEL_8B, TEXT_VOCAB, model_namespace, synthetic_layout, synthetic_tensors  # noqa: E402

PROMPTS = (40, 57, 23, 51)  # L = P + 2374 at 512x512 must stay within max_sequence_length = 2432


def gpu_info() -> dict:
    """Name, power limit, current and maximum SM clock of GPU 0 (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock, clock_max = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": clock, "sm_clock_max": clock_max}
    except Exception as e:  # the numbers are still printed; the card is then unknown
        return {"error": f"{type(e).__name__}: {e}"[:200]}


def build(device: str, max_batch: int, seed: int = 1000):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    m = LLaDAForMultiModalGeneration(model_namespace(MODEL_8B), max_seq_len=MODEL_8B["max_sequence_length"], max_batch=max_batch,
                                     device=device)
    for name, t in synthetic_tensors(MODEL_8B, device, seed):
        assert m.set_weight(name, t)
    m.load_state_dict({}, strict=True)
    torch.cuda.synchronize()
    return m


def requests(n: int, grid: int, device: str) -> list:
    from mmada_parallel_b200.schedule import cosine_schedule
    out = []
    for i in range(n):
        lay = synthetic_layout(seed=i, prompt_len=PROMPTS[i], grid=grid)
        out.append(dict(lay, noise_schedule=cosine_schedule, text_vocab_size=TEXT_VOCAB, codebook_size=CODEBOOK,
                        generator=torch.Generator(device=device).manual_seed(42 + i), **GEN))
    return out


def forward_flops(lens, rows_a, rows_b, window=None) -> float:
    """FLOP of one forward over sequences `lens` (packed, or one sequence) with rows_a text rows x V and rows_b image rows x the
    codebook. window = rows of the last block's row window (one sequence), None = the whole last block."""
    c = MODEL_8B
    d, ff, V, nl = c["d_model"], c["mlp_hidden_size"], c["vocab_size"], c["n_layers"]
    M = sum(lens)
    layer = 2.0 * M * d * (4 * d + 3 * ff) + 4.0 * d * sum(L * L for L in lens)
    f = (nl - 1) * layer
    if window is None:
        f += layer
    else:
        (L,) = lens
        f += 2.0 * M * d * 3 * d + 2.0 * window * d * (d + 3 * ff) + 4.0 * d * window * L
    return f + 2.0 * d * (rows_a * V + rows_b * CODEBOOK)


def sample_flops(reqs, batched: bool) -> float:
    """Executed FLOP of the requests' whole loops (the same forwards for both paths, except the sequential row windows)."""
    from mmada_parallel_b200.schedule import image_generation_step_indices
    total = 0.0
    for r in reqs:
        L = r["input_ids"].shape[1]
        n_text, n_img = r["text_end"] - r["text_start"], r["seq_len"]
        img_lo, img_hi = r["image_start"], r["image_start"] + n_img + n_img // r["newline_every"]
        use_win = not batched and L >= 1024
        win_text = n_text if use_win else None
        win_both = max(r["text_end"], img_hi) - min(r["text_start"], img_lo) if use_win else None
        win_img = img_hi - img_lo if use_win else None
        img_steps = set(image_generation_step_indices(r["text_steps"], r["timesteps"]))
        n_unc = int(r["cfg_scale"] != 0) + int(r["cfg_img"] != 0)
        for s in range(r["text_steps"]):
            if s in img_steps:
                total += forward_flops([L], n_text, n_img, win_both) + n_unc * forward_flops([L], 0, n_img, win_img)
            else:
                total += forward_flops([L], n_text, 0, win_text)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=1, help="timed repetitions of each (size, N) pair")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="32,16", help="VQ grids (32: 512x512, 16: 256x256)")
    ap.add_argument("--ns", default="1,2,4")
    ap.add_argument("--exact-grid", type=int, default=16, help="grid of the bit-exactness check with the splits off (0: skip)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch: needs a CUDA device (H100)")
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.generators.batch import generate_ti2ti_batch
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti

    device = "cuda:0"
    torch.cuda.set_device(device)
    ns = [int(x) for x in args.ns.split(",")]
    model = build(device, max_batch=max(ns))

    def run(reqs, batched):
        torch.manual_seed(1234)  # still-masked image tokens are drawn from the global CPU RNG after the loop
        with contextlib.redirect_stdout(io.StringIO()):
            return generate_ti2ti_batch(model, reqs) if batched else [generate_ti2ti(model, **r) for r in reqs]

    def timed(reqs, batched):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = run(reqs, batched)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def n_diff(a, b):
        return sum(sum(x != y for x, y in zip(ra[0], rb[0])) + sum(x != y for x, y in zip(ra[1], rb[1])) for ra, rb in zip(a, b))

    res = {"metric": "packed_batch_vs_sequential_tokens_per_s", "model": "8B synthetic (bench.py), bf16",
           "prompts": list(PROMPTS), "gen": {k: GEN[k] for k in ("text_steps", "timesteps", "cfg_scale", "cfg_img")}, "runs": []}
    t_start = time.time()
    with torch.no_grad():
        for grid in (int(x) for x in args.sizes.split(",")):
            for _ in range(args.warmup):
                run(requests(1, grid, device), True)
                run(requests(1, grid, device), False)
            for n in ns:
                tokens = n * (grid * grid + GEN["text_gen_length"])
                ms = {True: [], False: []}
                outs = {}
                for rep in range(args.reps):
                    for batched in ((True, False) if rep % 2 == 0 else (False, True)):  # alternating order
                        t, outs[batched] = timed(requests(n, grid, device), batched)
                        ms[batched].append(t)
                reqs = requests(n, grid, device)
                row = {"image": f"{grid * 16}x{grid * 16}", "n": n, "lengths": [r["input_ids"].shape[1] for r in reqs]}
                for batched, key in ((True, "batch"), (False, "sequential")):
                    mean = sum(ms[batched]) / len(ms[batched])
                    fl = sample_flops(reqs, batched)
                    row[key] = {"ms": [round(v, 1) for v in ms[batched]], "tokens_per_s": round(tokens / (mean / 1e3), 2),
                                "pflop": round(fl / 1e15, 3), "tflops": round(fl / (mean / 1e3) / 1e12, 1)}
                row["ratio_batch_over_sequential"] = round(row["batch"]["tokens_per_s"] / row["sequential"]["tokens_per_s"], 4)
                row["differing_ids_default_options"] = n_diff(outs[True], outs[False])
                row["total_ids"] = sum(len(r[0]) + len(r[1]) for r in outs[False])
                res["runs"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
        if args.exact_grid:
            n = max(ns)
            _lib.lib.mmdp_set_gemm_splitk(0)
            _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 0))
            try:
                b = run(requests(n, args.exact_grid, device), True)
                s = run(requests(n, args.exact_grid, device), False)
            finally:
                _lib.lib.mmdp_set_gemm_splitk(2)
                _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))
            res["exact_splits_off"] = {"image": f"{args.exact_grid * 16}x{args.exact_grid * 16}", "n": n, "ids_equal": b == s,
                                       "differing_ids": n_diff(b, s)}
    res["gpu"] = gpu_info()
    res["wall_s"] = round(time.time() - t_start, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
