"""Tensor-parallel grouped-query attention and the q/k/v bias: the 8B shapes of bench.py (d = 4096, 32 heads, 32 layers,
ff = 12288, L = 2414) sharded over tp in {2, 4, 8} ranks, with n_kv_heads in {32, 8, 1}, each without and with a q/k/v bias.

On one GPU, per configuration and per rank (tensor_parallel.kv_shard decides the rank's kv heads), timed with CUDA events:
  qkv        the rank's QKV projection + RoPE + V^T launch (mmdp_qkv_rope_tp for the multi-head shard without a bias, else
             mmdp_qkv_rope_tp_gqa), 20 calls;
  attention  the rank's attention launches (mmdp_attention / mmdp_attention_gqa, B = 1), 20 calls;
  sim_rank   one forward of the 32 layers issued op by op for all tp simulated ranks on one stream (the sequence of
             mmdp_tp_forward: QKV, attention, attn_out pushed to the owners' receive buffers, reduce + residual + norm +
             broadcast, SwiGLU, ff_out pushed, reduce), divided by tp. Every layer reuses one layer's shard weights (the times
             depend on the shapes only). The ranks' NVLink traffic becomes local stores, and every reduce call is preceded by the
             small fills that set the flags it waits on, so this is a per-rank compute time, not the time of a real TP forward.
Under torchrun with >= 2 GPUs (tp = world size) it also times whole 512x512 samples of bench.py's workload through
generate_ti2ti with TensorParallelLLaDA (--steps samples after --warmup); with one GPU those are printed as "not measured".
The GPU's name, power limit and SM clock are read in the same run. Prints one JSON line.

    python tools/bench_tp_gqa.py [--out FILE]
    torchrun --nproc-per-node 8 tools/bench_tp_gqa.py --steps 1 --warmup 0
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes as C
import io
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import CODEBOOK, GEN, MODEL_8B, TEXT_VOCAB, model_namespace, synthetic_layout  # noqa: E402
from tools.bench_gqa import gpu_info, time_op  # noqa: E402

L = 2414
TPS, KV_HEADS = (2, 4, 8), (32, 8, 1)


class Rank:
    """One simulated rank's layer shard, buffers and peer-visible state (see tests/test_gpu_tp_ops.py, SimRanks)."""

    def __init__(self, tp, r, n_kv, bias, g, dev):
        from mmada_parallel_b200.tensor_parallel import kv_shard
        d, ff, H = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["n_heads"]
        self.Hl, self.Hkv = H // tp, kv_shard(H, n_kv, r, tp)[1]
        self.gqa = self.Hkv != self.Hl or bias
        da, dkv, ffl = self.Hl * 128, self.Hkv * 128, ff // tp

        def mk(*shape):
            return (torch.randn(*shape, device=dev, generator=g) * 0.02).to(torch.bfloat16)

        self.wqkv, self.wo, self.w13, self.w2 = mk(da + 2 * dkv, d), mk(d, da), mk(2 * ffl, d), mk(d, ffl)
        self.bqkv = mk(da + 2 * dkv) if bias else None
        self.norm = torch.ones(d, dtype=torch.bfloat16, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.q, self.att, self.k = torch.empty(L, da, **bf), torch.empty(L, da, **bf), torch.empty(L, dkv, **bf)
        self.h = torch.empty(L, ffl, **bf)
        self.vt = torch.zeros(1, self.Hkv, 128, (L + 7) // 8 * 8, **bf)
        R = (L + tp - 1) // tp
        self.xn = torch.zeros(L, d, **bf)
        self.x = torch.zeros(R, d, **bf)
        self.flags = torch.zeros(2, 8, dtype=torch.int32, device=dev)
        self.done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.recv = [torch.zeros(tp, R, d, dtype=torch.float32, device=dev) for _ in range(2)]

    def qkv(self, cos, sin, s):
        from mmada_parallel_b200._lib import check, lib
        d, Lpad = MODEL_8B["d_model"], self.vt.shape[-1]
        if self.gqa:
            check(lib.mmdp_qkv_rope_tp_gqa(self.xn.data_ptr(), d, self.wqkv.data_ptr(), None if self.bqkv is None else self.bqkv.data_ptr(),
                                           L, d, self.Hl, self.Hkv, L, Lpad, cos.data_ptr(), sin.data_ptr(), self.q.data_ptr(),
                                           self.k.data_ptr(), self.vt.data_ptr(), s))
        else:
            check(lib.mmdp_qkv_rope_tp(self.xn.data_ptr(), d, self.wqkv.data_ptr(), L, d, self.Hl, L, Lpad, cos.data_ptr(), sin.data_ptr(),
                                       self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), s))

    def attention(self, s):
        from mmada_parallel_b200._lib import check, lib
        Lpad, scale = self.vt.shape[-1], 1.0 / math.sqrt(128.0)
        if self.gqa:
            check(lib.mmdp_attention_gqa(self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), self.att.data_ptr(), 1, None, self.Hl,
                                         self.Hkv, L, Lpad, scale, s))
        else:
            check(lib.mmdp_attention(self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), self.att.data_ptr(), 1, self.Hl, L, Lpad,
                                     scale, s))


def sim_forward(ranks, cos, sin, n_layers, epoch):
    """One forward of n_layers issued for every simulated rank in turn (the order of tests/test_gpu_tp_ops.py::sim_tp_forward).
    Before each reduce call every flag it waits on already holds the call's epoch. Returns the last epoch used."""
    from mmada_parallel_b200._lib import EPI_SWIGLU, check, lib, stream_ptr
    tp, d, s = len(ranks), MODEL_8B["d_model"], stream_ptr()
    R = (L + tp - 1) // tp
    xn_arr = (C.c_void_p * tp)(*[rk.xn.data_ptr() for rk in ranks])
    fl_arr = (C.c_void_p * tp)(*[rk.flags.data_ptr() for rk in ranks])
    recv_arr = [(C.c_void_p * tp)(*[rk.recv[b].data_ptr() for rk in ranks]) for b in range(2)]

    def reduce_all(n_src, buf, ep):
        for my, rk in enumerate(ranks):
            rk.flags.fill_(ep)  # the call waits on its own flag array only
            r0 = my * R
            check(lib.mmdp_tp_reduce_norm(rk.recv[buf].data_ptr() if n_src else None, R, n_src, xn_arr, fl_arr, tp, my, rk.x.data_ptr(),
                                          rk.norm.data_ptr(), r0, min(R, L - r0), d, 1e-5, ep & 0xFFFFFFFF, rk.done.data_ptr(), s))

    epoch += 1
    reduce_all(0, 0, epoch)
    for _ in range(n_layers):
        for my, rk in enumerate(ranks):
            rk.qkv(cos, sin, s)
            rk.attention(s)
            da = rk.q.shape[1]
            check(lib.mmdp_gemm_f32_scatter(rk.att.data_ptr(), da, rk.wo.data_ptr(), da, L, d, da, recv_arr[0], tp, R, my, s))
        epoch += 1
        reduce_all(tp, 0, epoch)
        for my, rk in enumerate(ranks):
            ffl = rk.h.shape[1]
            check(lib.mmdp_gemm_bf16(EPI_SWIGLU, rk.xn.data_ptr(), d, rk.w13.data_ptr(), d, L, 2 * ffl, d, rk.h.data_ptr(), ffl, None, 0, s))
            check(lib.mmdp_gemm_f32_scatter(rk.h.data_ptr(), ffl, rk.w2.data_ptr(), ffl, L, d, ffl, recv_arr[1], tp, R, my, s))
        epoch += 1
        reduce_all(tp, 1, epoch)
    return epoch


def one_gpu(dev):
    from mmada_parallel_b200.model import rope_tables
    cos, sin = (t.to(dev) for t in rope_tables(128, 500000.0, L))
    g = torch.Generator(device=dev).manual_seed(0)
    results = []
    for tp in TPS:
        for n_kv in KV_HEADS:
            for bias in (False, True):
                ranks = [Rank(tp, r, n_kv, bias, g, dev) for r in range(tp)]
                for rk in ranks:
                    rk.xn.normal_(0.0, 1.0, generator=g)
                    rk.x.normal_(0.0, 1.0, generator=g)
                rk0 = ranks[0]
                t_qkv = time_op(lambda: rk0.qkv(cos, sin, None))
                t_attn = time_op(lambda: rk0.attention(None))
                epoch = [sim_forward(ranks, cos, sin, MODEL_8B["n_layers"], 0)]  # warm-up
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                reps = 2
                e0.record()
                for _ in range(reps):
                    epoch[0] = sim_forward(ranks, cos, sin, MODEL_8B["n_layers"], epoch[0])
                e1.record()
                torch.cuda.synchronize()
                t_sim = e0.elapsed_time(e1) / reps / tp
                r = {"tp": tp, "n_kv_heads": n_kv, "qkv_bias": bias, "kv_heads_per_rank": rk0.Hkv,
                     "kv_replicated_on": tp // n_kv if n_kv < tp else 1, "qkv_N": rk0.wqkv.shape[0],
                     "qkv_ms": round(t_qkv, 4), "attention_ms": round(t_attn, 4), "sim_rank_forward_ms": round(t_sim, 2)}
                print(json.dumps(r), file=sys.stderr, flush=True)
                results.append(r)
                del ranks, rk0
                torch.cuda.empty_cache()
    return results


def synthetic_state_dict(n_kv, bias, dev, seed=1000):
    """bench.py's synthetic 8B tensors with n_kv kv heads and, optionally, q/k/v biases (the same on every rank)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    d, ff, V, dkv = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["vocab_size"], 128 * n_kv

    def mk(*shape, ones=False):
        if ones:
            return torch.ones(shape, dtype=torch.bfloat16, device=dev)
        return torch.empty(shape, dtype=torch.bfloat16, device=dev).normal_(0.0, 0.02, generator=g)

    sd = {"model.transformer.wte.weight": mk(V, d), "model.transformer.ff_out.weight": mk(V, d), "model.transformer.ln_f.weight": mk(d, ones=True)}
    for i in range(MODEL_8B["n_layers"]):
        p = f"model.transformer.blocks.{i}."
        for n, shape in (("q_proj", (d, d)), ("k_proj", (dkv, d)), ("v_proj", (dkv, d)), ("attn_out", (d, d)), ("ff_proj", (ff, d)),
                         ("up_proj", (ff, d)), ("ff_out", (d, ff))):
            sd[p + n + ".weight"] = mk(*shape)
        for n in ("attn_norm", "ff_norm"):
            sd[p + n + ".weight"] = mk(d, ones=True)
        if bias:
            for n, rows in (("q_proj", d), ("k_proj", dkv), ("v_proj", dkv)):
                sd[p + n + ".bias"] = mk(rows)
    return sd


def multi_gpu_samples(args, rank, world, dev):
    """Whole 512x512 samples through generate_ti2ti on a TP = world model, per kv-head count and bias."""
    import torch.distributed as dist
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    lay = synthetic_layout(seed=0)
    kw = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    out = []
    for n_kv in KV_HEADS:
        for bias in (False, True):
            if n_kv % world and world % n_kv:
                out.append({"tp": world, "n_kv_heads": n_kv, "qkv_bias": bias, "sample_s": "not supported (tp and n_kv_heads)"})
                continue
            cfg = model_namespace(MODEL_8B)
            cfg.n_kv_heads, cfg.include_qkv_bias = n_kv, bias
            sd = synthetic_state_dict(n_kv, bias, dev)
            m = TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=MODEL_8B["max_sequence_length"], device=dev, text_vocab_size=TEXT_VOCAB,
                                    codebook_size=CODEBOOK)
            del sd
            torch.cuda.empty_cache()
            times = []
            for i in range(args.warmup + args.steps):
                dist.barrier()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                with contextlib.redirect_stdout(io.StringIO()):
                    torch.manual_seed(5)
                    generate_ti2ti(m, lay["input_ids"], generator=torch.Generator(device=dev).manual_seed(42), **kw, **GEN)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times.append(round(e0.elapsed_time(e1) / 1e3, 3))
            dist.barrier()
            del m
            torch.cuda.empty_cache()
            out.append({"tp": world, "n_kv_heads": n_kv, "qkv_bias": bias, "sample_s": times})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1, help="timed samples per configuration under torchrun with >= 2 GPUs")
    ap.add_argument("--warmup", type=int, default=0, help="untimed samples per configuration first")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tp_gqa: needs a CUDA device (H100)")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}"
    torch.cuda.set_device(dev)
    line = {"gpu": gpu_info(), "L": L, "model": "8B synthetic (bench.py shapes)"}
    with torch.no_grad():
        if world >= 2:
            import torch.distributed as dist
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
            line["samples"] = multi_gpu_samples(args, rank, world, dev)
            dist.destroy_process_group()
            if rank != 0:
                return
        else:
            line["samples"] = "not measured (needs torchrun with >= 2 GPUs)"
            line["per_rank"] = one_gpu(dev)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
