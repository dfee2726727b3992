"""The bf16 GEMM launches of one 8B sample, each at its production epilogue, timed with CUDA events after warm-up, and the
per-tile fixed cost of the persistent kernel. Prints one JSON line. The GPU's name, power limit and maximum SM clock are read
in the same run (nvidia-smi query).

    python tools/bench_gemm.py [--reps 20] [--out FILE]

Per-tile fixed cost: with the split-K tail off every CTA runs whole tiles, so a launch takes t(K) = waves * (K/64 * c + x),
where c is the main-loop time of one 64-deep k-block and x what a tile costs beyond its main loop (the epilogue and whatever
the pipeline cannot hide at a tile boundary). Timing the same M x N at K = 4096 and K = 12288 gives
x = (3 * t(4096) - t(12288)) / (2 * waves). QKV + RoPE takes the same fit: N = 12288 (32 heads) at both K.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import CODEBOOK, MODEL_8B  # noqa: E402
from tools.bench_fp8 import L_SAMPLE, gpu_info, time_op  # noqa: E402

WINDOW_M = (256, 1056, 1313)  # rows of the last block's windowed forwards


def waves_no_split(M: int, N: int, epi: int, sms: int) -> int:
    """Waves of the plan gemm.cu picks with the split-K tail off (tile width 256 or 192 by the same cost model)."""
    from mmada_parallel_b200 import _lib
    best = None
    for bn in ((256, 192) if epi in (_lib.EPI_PLAIN, _lib.EPI_RESID, _lib.EPI_F32) else (256,)):
        tiles = -(-M // 128) * -(-N // bn)
        waves = -(-tiles // sms)
        cost = waves * bn * (1.04 if bn == 192 else 1.0)
        if best is None or cost < best[0]:
            best = (cost, waves)
    return best[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="timed calls per launch shape")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm: needs a CUDA device (H100)")
    from mmada_parallel_b200 import _lib

    device = "cuda:0"
    torch.cuda.set_device(device)
    info = gpu_info()
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    d, ff, H, V = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["n_heads"], MODEL_8B["vocab_size"]
    g = torch.Generator(device=device).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device=device, generator=g) * scale).to(torch.bfloat16)

    xa = {K: rnd(L_SAMPLE, K, scale=0.5) for K in (d, ff)}  # activations, contiguous rows as in the forward
    weights = {}

    def w(N, K):
        if (N, K) not in weights:
            weights[(N, K)] = rnd(N, K, scale=0.02)
        return weights[(N, K)]

    resid = rnd(L_SAMPLE, d)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, device=device, dtype=torch.float32) / 128))
    ang = torch.arange(L_SAMPLE, device=device, dtype=torch.float32)[:, None] * inv[None, :]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()

    def entry(M, N, K, ms):
        return {"M": M, "N": N, "K": K, "ms": round(ms, 4), "tflops": round(2.0 * M * N * K / ms / 1e9, 1)}

    launches = {}
    with torch.no_grad():
        M = L_SAMPLE
        # q, k and V^T are allocated once (the forward's buffers are too), so only the GEMM launch is timed
        q = torch.empty(M, d, dtype=torch.bfloat16, device=device)
        k = torch.empty_like(q)
        vt = torch.zeros(1, H, 128, -(-M // 8) * 8, dtype=torch.bfloat16, device=device)

        def qkv(K):
            """QKV + RoPE of H heads (N = 3 * 128 H) over K input columns: the tensor-parallel entry takes K apart from H."""
            _lib.check(_lib.lib.mmdp_qkv_rope_tp(_lib.ptr(xa[K]), K, _lib.ptr(w(3 * d, K)), M, K, H, M, vt.shape[-1], _lib.ptr(cos),
                                                 _lib.ptr(sin), _lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.stream_ptr()))

        launches["qkv_rope"] = entry(M, 3 * d, d, time_op(lambda: qkv(d), args.reps))
        for m in (M,) + WINDOW_M:
            sfx = "" if m == M else f"_m{m}"
            r = resid[:m]
            launches["attn_out_resid" + sfx] = entry(m, d, d, time_op(
                lambda: _lib.gemm_bf16(xa[d][:m], w(d, d), _lib.EPI_RESID, resid=r, out=r), args.reps))
            launches["gate_up_swiglu" + sfx] = entry(m, 2 * ff, d, time_op(
                lambda: _lib.gemm_bf16(xa[d][:m], w(2 * ff, d), _lib.EPI_SWIGLU), args.reps))
            launches["ff_out_resid" + sfx] = entry(m, d, ff, time_op(
                lambda: _lib.gemm_bf16(xa[ff][:m], w(d, ff), _lib.EPI_RESID, resid=r, out=r), args.reps))
        launches["text_head"] = entry(256, V, d, time_op(lambda: _lib.gemm_bf16(xa[d][:256], w(V, d)), args.reps))
        launches["image_head"] = entry(1024, CODEBOOK, d, time_op(lambda: _lib.gemm_bf16(xa[d][:1024], w(CODEBOOK, d)), args.reps))

        per_tile = {}
        _lib.lib.mmdp_set_gemm_splitk(0)
        try:
            for name, N, epi in (("plain", 3 * d, _lib.EPI_PLAIN), ("resid", d, _lib.EPI_RESID), ("swiglu", 2 * ff, _lib.EPI_SWIGLU),
                                 ("qkv_rope", 3 * d, None)):
                t = {}
                for K in (d, ff):
                    r = resid[:M] if epi == _lib.EPI_RESID else None
                    if epi is None:
                        t[K] = time_op(lambda: qkv(K), args.reps)
                    else:
                        t[K] = time_op(lambda: _lib.gemm_bf16(xa[K][:M], w(N, K), epi, resid=r, out=r), args.reps)
                waves = waves_no_split(M, N, epi, sms)
                x_ms = (3 * t[d] - t[ff]) / (2 * waves)
                loop_ms = t[d] / waves - x_ms  # main loop of one K = 4096 tile
                per_tile[name] = {"M": M, "N": N, "waves": waves, "ms_k4096": round(t[d], 4), "ms_k12288": round(t[ff], 4),
                                  "x_us": round(1e3 * x_ms, 2), "mainloop_k4096_us": round(1e3 * loop_ms, 2),
                                  "x_share_of_k4096_tile": round(x_ms / (t[d] / waves), 4)}
        finally:
            _lib.lib.mmdp_set_gemm_splitk(2)
    res = {"metric": "gemm_bf16_by_launch", "gpu": info, "sms": sms, "reps": args.reps, "launches": launches,
           "per_tile_fixed_cost_splitk_off": per_tile}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
