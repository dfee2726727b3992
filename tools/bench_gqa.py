"""Grouped-query attention and the q/k/v bias on one GPU: the 8B shapes of bench.py (d = 4096, 32 heads, 32 layers, L = 2414) with
n_kv_heads in {32, 8, 1}, each without and with a q/k/v bias. Per configuration, timed with CUDA events:
  qkv        the QKV projection + RoPE + V^T launch (mmdp_qkv_rope_gqa, N = d + 2 * 128 * n_kv_heads);
  attention  the attention launches of one block (mmdp_attention_gqa, B = 1);
  forward    one forward of the whole model with the sample's restricted head (text rows x V, image rows x the codebook);
  sample     whole 512x512@64 samples of bench.py's denoise loop (--steps, after --warmup).
FLOPs are computed from the shapes. The GPU's name, power limit and SM clock are read in the same run. Prints one JSON line.

    python tools/bench_gqa.py --steps 1 --warmup 0 [--out FILE]
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

from bench import CODEBOOK, GEN, MODEL_8B, TEXT_VOCAB, model_namespace, synthetic_layout  # noqa: E402

L_SAMPLE = 2414  # sequence length of the synthetic layout (prompt 40)


def gpu_info() -> dict:
    """Name, power limit, current and maximum SM clock of GPU 0 (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock, clock_max = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": clock, "sm_clock_max": clock_max}
    except Exception as e:  # the numbers are still printed; the card is then unknown
        return {"error": f"{type(e).__name__}: {e}"[:200]}


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


def build(n_kv: int, bias: bool, device: str, seed: int = 1000):
    """The bench.py 8B model (normal(0, 0.02) matrices, unit norms) with n_kv kv heads and, optionally, q/k/v biases."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    cfg = model_namespace(MODEL_8B)
    cfg.n_kv_heads, cfg.include_qkv_bias = n_kv, bias
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=MODEL_8B["max_sequence_length"], max_batch=1, device=device)
    g = torch.Generator(device=device).manual_seed(seed)
    d, ff, V, dkv = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["vocab_size"], 128 * n_kv

    def mk(*shape, ones=False):
        if ones:
            return torch.ones(shape, dtype=torch.bfloat16, device=device)
        return torch.empty(shape, dtype=torch.bfloat16, device=device).normal_(0.0, 0.02, generator=g)

    sd = {"model.transformer.wte.weight": mk(V, d), "model.transformer.ff_out.weight": mk(V, d),
          "model.transformer.ln_f.weight": mk(d, ones=True)}
    for name, t in sd.items():
        m.set_weight(name, t)
    for i in range(MODEL_8B["n_layers"]):
        p = f"model.transformer.blocks.{i}."
        for n, shape in (("q_proj", (d, d)), ("k_proj", (dkv, d)), ("v_proj", (dkv, d)), ("attn_out", (d, d)), ("ff_proj", (ff, d)),
                         ("up_proj", (ff, d)), ("ff_out", (d, ff))):
            m.set_weight(p + n + ".weight", mk(*shape))
        for n in ("attn_norm", "ff_norm"):
            m.set_weight(p + n + ".weight", mk(d, ones=True))
        if bias:
            for n, rows in (("q_proj", d), ("k_proj", dkv), ("v_proj", dkv)):
                m.set_weight(p + n + ".bias", mk(rows))
    m.load_state_dict({}, strict=True)
    torch.cuda.synchronize()
    return m


def flops(n_kv: int, n_text: int, n_img: int) -> dict:
    d, ff, V, H, nl, L = (MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["vocab_size"], MODEL_8B["n_heads"],
                          MODEL_8B["n_layers"], L_SAMPLE)
    qkv = 2.0 * L * (d + 2 * 128 * n_kv) * d
    attn = 4.0 * H * L * L * 128
    layer = qkv + attn + 2.0 * L * d * d + 2.0 * L * 2 * ff * d + 2.0 * L * ff * d
    head = 2.0 * d * (n_text * V + n_img * CODEBOOK)
    return {"qkv": qkv, "attention": attn, "forward": nl * layer + head}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1, help="timed samples per configuration (0: no sample)")
    ap.add_argument("--warmup", type=int, default=0, help="untimed samples per configuration first")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gqa: needs a CUDA device (H100)")
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.generators.parallel_generator import DenoiseState, denoise_loop
    from mmada_parallel_b200.model import rope_tables
    from mmada_parallel_b200.schedule import cosine_schedule

    device = "cuda:0"
    torch.cuda.set_device(device)
    info = gpu_info()
    lay = synthetic_layout(seed=0)
    pos_args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every")}
    loop_kw = dict(text_steps=GEN["text_steps"], timesteps=GEN["timesteps"], temperature=GEN["temperature"],
                   text_temperature=GEN["text_temperature"], cfg_scale=GEN["cfg_scale"], cfg_img=GEN["cfg_img"],
                   noise_schedule=cosine_schedule, text_vocab_size=TEXT_VOCAB, codebook_size=CODEBOOK)
    ids = lay["input_ids"].to(device)
    ts, te, s0, grid = lay["text_start"], lay["text_end"], lay["image_start"], lay["newline_every"]
    text_rows = torch.arange(ts, te, dtype=torch.int32, device=device)
    img_rows = torch.tensor([s0 + r * (grid + 1) + c for r in range(grid) for c in range(grid)], dtype=torch.int32, device=device)
    d, H, L = MODEL_8B["d_model"], MODEL_8B["n_heads"], L_SAMPLE
    cos, sin = (t.to(device) for t in rope_tables(128, 500000.0, L))
    g = torch.Generator(device=device).manual_seed(0)
    a = (torch.randn(L, d, device=device, generator=g) * 0.5).to(torch.bfloat16)
    results = []
    with torch.no_grad():
        for n_kv in (32, 8, 1):
            for bias in (False, True):
                dkv = 128 * n_kv
                w = (torch.randn(d + 2 * dkv, d, device=device, generator=g) * 0.02).to(torch.bfloat16)
                b = (torch.randn(d + 2 * dkv, device=device, generator=g) * 0.02).to(torch.bfloat16) if bias else None
                fl = flops(n_kv, len(text_rows), len(img_rows))
                if n_kv == H and not bias:  # the multi-head launch the model runs for this config
                    t_qkv = time_op(lambda: _lib.qkv_rope(a, w, H, L, cos, sin))
                else:
                    t_qkv = time_op(lambda: _lib.qkv_rope_gqa(a, w, b, H, n_kv, L, cos, sin))
                q, k, vt = _lib.qkv_rope_gqa(a, w, b, H, n_kv, L, cos, sin)
                t_attn = time_op(lambda: _lib.attention_gqa(q, k, vt, H, n_kv, 128 ** -0.5, B=1, L=L))
                del q, k, vt, w, b
                m = build(n_kv, bias, device)
                t_fwd = time_op(lambda: m.forward_rows(ids, rows_a=text_rows, rows_b=img_rows, col0_b=TEXT_VOCAB, ncols_b=CODEBOOK),
                                reps=5)
                sample_s = []
                rng = torch.Generator(device=device).manual_seed(42)
                for i in range(args.warmup + args.steps):
                    st = DenoiseState(m, lay["input_ids"], uncon_text=lay["uncon_text"], uncon_image=lay["uncon_image"],
                                      cfg_scale=GEN["cfg_scale"], cfg_img=GEN["cfg_img"], codebook_size=CODEBOOK, **pos_args)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    e0.record()
                    denoise_loop(st, generator=rng, **loop_kw)
                    e1.record()
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        sample_s.append(round(e0.elapsed_time(e1) / 1e3, 3))
                del m
                torch.cuda.empty_cache()
                r = {"n_kv_heads": n_kv, "qkv_bias": bias, "qkv_N": d + 2 * dkv,
                     "qkv_ms": round(t_qkv, 4), "qkv_tflops": round(fl["qkv"] / t_qkv / 1e9, 1),
                     "attention_ms": round(t_attn, 4), "attention_tflops": round(fl["attention"] / t_attn / 1e9, 1),
                     "forward_ms": round(t_fwd, 2), "forward_tflops": round(fl["forward"] / t_fwd / 1e9, 1),
                     "sample_s": sample_s}
                print(json.dumps(r), file=sys.stderr, flush=True)
                results.append(r)
    line = json.dumps({"gpu": info, "L": L, "model": "8B synthetic (bench.py shapes)", "results": results})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
