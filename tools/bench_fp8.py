"""FP8 vs bf16 on one GPU: the 8B synthetic model of bench.py built twice (precision "bf16" and "fp8", same seeded weights),
K whole 512x512@64 samples (bench.py's denoise loop and settings) timed with CUDA events, alternating the two models in one
process, one profiled sample each (time and work per launch kind, and from their difference the quantiser's time per forward),
the e4m3 and bf16 GEMMs of the block shapes on their own, and the FP8-vs-bf16 deviation of the first step's logits. Prints one
JSON line. The GPU's name and power limit are read in the same run (nvidia-smi query).

    python tools/bench_fp8.py --steps 2 --warmup 1 [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import (CODEBOOK, GEN, MODEL_8B, TEXT_VOCAB, TOKENS_PER_SAMPLE, model_namespace,  # noqa: E402
                   synthetic_layout, synthetic_tensors)

L_SAMPLE = 2414  # sequence length of the synthetic layout (prompt 40)


def gpu_info() -> dict:
    """Name, power limit and maximum SM clock of GPU 0 (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # the numbers are still printed; the card is then unknown
        return {"error": f"{type(e).__name__}: {e}"[:200]}


def build(precision: str, device: str, seed: int = 1000):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    m = LLaDAForMultiModalGeneration(model_namespace(MODEL_8B), max_seq_len=MODEL_8B["max_sequence_length"], max_batch=1,
                                     device=device, precision=precision)
    for name, t in synthetic_tensors(MODEL_8B, device, seed):
        assert m.set_weight(name, t)
    m.load_state_dict({}, strict=True)
    torch.cuda.synchronize()
    return m


def time_op(fn, reps: int = 20) -> float:
    """Milliseconds per call (CUDA events around `reps` calls after two warm-up calls)."""
    fn(); fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gemm_table(device: str) -> dict:
    """The block GEMMs of one 8B layer at L = 2414 (QKV, attn_out, gate/up + SwiGLU, ff_out), e4m3 against bf16 kernels. (The
    quantiser is timed from the profiled samples instead: its launches of 15-45 us are shorter than a Python call.)"""
    from mmada_parallel_b200 import _lib
    g = torch.Generator(device=device).manual_seed(0)
    out = {}
    d, ff, M = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], L_SAMPLE
    for name, N, K, epi in (("qkv", 3 * d, d, _lib.EPI_PLAIN), ("attn_out", d, d, _lib.EPI_RESID),
                            ("w13_swiglu", 2 * ff, d, _lib.EPI_SWIGLU), ("ff_out", d, ff, _lib.EPI_RESID)):
        a = (torch.randn(M, K, device=device, generator=g) * 0.5).to(torch.bfloat16)
        w = (torch.randn(N, K, device=device, generator=g) * 0.02).to(torch.bfloat16)
        r = torch.randn(M, N, device=device, generator=g).to(torch.bfloat16) if epi == _lib.EPI_RESID else None
        qa, sa = _lib.quantize_fp8(a, 128)
        qw, sw = _lib.quantize_fp8(w, K)
        sw = sw[0].contiguous()
        flops = 2.0 * M * N * K
        t8 = time_op(lambda: _lib.gemm_fp8(qa, sa, qw, sw, epi, resid=r))
        t16 = time_op(lambda: _lib.gemm_bf16(a, w, epi, resid=r))
        out[name] = {"M": M, "N": N, "K": K, "fp8_ms": round(t8, 4), "fp8_tflops": round(flops / t8 / 1e9, 1),
                     "bf16_ms": round(t16, 4), "bf16_tflops": round(flops / t16 / 1e9, 1)}
    return out


def first_step_deviation(m16, m8, lay: dict, device: str) -> dict:
    """One forward on the sample's first-step ids: text rows x all columns, image rows x the codebook window."""
    ids = lay["input_ids"].to(device)
    ts, te, s0, grid = lay["text_start"], lay["text_end"], lay["image_start"], lay["newline_every"]
    text_rows = torch.arange(ts, te, dtype=torch.int32, device=device)
    img_rows = torch.tensor([s0 + r * (grid + 1) + c for r in range(grid) for c in range(grid)], dtype=torch.int32, device=device)
    res = {}
    outs = [m.forward_rows(ids, rows_a=text_rows, rows_b=img_rows, col0_b=TEXT_VOCAB, ncols_b=CODEBOOK) for m in (m16, m8)]
    for i, what in enumerate(("text", "codebook")):
        ref, got = outs[0][i].float(), outs[1][i].float()
        err = got - ref
        res[what] = {"rel_rms": round((err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item(), 5),
                     "max_abs_err": round(err.abs().max().item(), 5), "scale": round(ref.abs().max().item(), 5),
                     "argmax_equal": round((got.argmax(-1) == ref.argmax(-1)).float().mean().item(), 5)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="timed samples per precision")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8: needs a CUDA device (H100)")
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.generators.parallel_generator import DenoiseState, denoise_loop
    from mmada_parallel_b200.schedule import cosine_schedule

    device = "cuda:0"
    torch.cuda.set_device(device)
    info = gpu_info()
    models = {p: build(p, device) for p in ("bf16", "fp8")}
    lay = synthetic_layout(seed=0)
    pos_args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every")}
    loop_kw = dict(text_steps=GEN["text_steps"], timesteps=GEN["timesteps"], temperature=GEN["temperature"],
                   text_temperature=GEN["text_temperature"], cfg_scale=GEN["cfg_scale"], cfg_img=GEN["cfg_img"],
                   noise_schedule=cosine_schedule, text_vocab_size=TEXT_VOCAB, codebook_size=CODEBOOK)

    def sample(m, rng):
        st = DenoiseState(m, lay["input_ids"], uncon_text=lay["uncon_text"], uncon_image=lay["uncon_image"], cfg_scale=GEN["cfg_scale"],
                          cfg_img=GEN["cfg_img"], codebook_size=CODEBOOK, **pos_args)
        return denoise_loop(st, generator=rng, **loop_kw)

    rngs = {p: torch.Generator(device=device).manual_seed(42) for p in models}
    with torch.no_grad():
        dev = first_step_deviation(models["bf16"], models["fp8"], lay, device)
        for _ in range(args.warmup):
            for p, m in models.items():
                sample(m, rngs[p])
        ms = {p: [] for p in models}
        for _ in range(args.steps):
            for p, m in models.items():  # alternating: both see the same clocks and neighbours
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                sample(m, rngs[p])
                e1.record()
                torch.cuda.synchronize()
                ms[p].append(e0.elapsed_time(e1))
        prof = {}
        for p, m in models.items():
            _lib.lib.mmdp_prof_enable(1)
            sample(m, rngs[p])
            s = _lib.prof_summary()
            _lib.lib.mmdp_prof_enable(0)
            prof[p] = {k: {"ms": round(v[0], 1), "launches": v[2],
                           ("tflops" if k in ("gemm", "attention") else "gbytes_per_s"): round(v[1] / max(v[0], 1e-9) / 1e9, 1)}
                       for k, v in s.items()}
        gemms = gemm_table(device)
    res = {"metric": "fp8_vs_bf16_tokens_per_s", "gpu": info, "model": "8B synthetic, 512x512@64 + 256 text tokens, L=2414",
           "samples_per_precision": args.steps}
    for p in models:
        mean_ms = sum(ms[p]) / len(ms[p])
        res[p] = {"sample_ms": [round(v, 1) for v in ms[p]], "tokens_per_s": round(TOKENS_PER_SAMPLE / (mean_ms / 1e3), 2),
                  "profile": prof[p]}
    res["speedup_fp8"] = round(res["fp8"]["tokens_per_s"] / res["bf16"]["tokens_per_s"], 4)
    # the quantiser is the FP8 sample's only extra row-kernel work: 4 launches per layer and forward (xn twice, att, h)
    extra = prof["fp8"]["row"]["launches"] - prof["bf16"]["row"]["launches"]
    forwards = extra / (4 * MODEL_8B["n_layers"])
    q_ms = (prof["fp8"]["row"]["ms"] - prof["bf16"]["row"]["ms"]) / forwards
    d, ff = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"]
    q_bytes = MODEL_8B["n_layers"] * L_SAMPLE * (3 * d + ff) * 3  # bf16 read + e4m3 written (scales: 1/64 more)
    res["quantize_per_forward"] = {"ms": round(q_ms, 3), "forwards_per_sample": forwards, "tb_per_s": round(q_bytes / q_ms / 1e9, 2)}
    res["gemm_by_shape"] = gemms
    res["first_step_logit_deviation"] = dev
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
