"""FP8 (e4m3) block linears under tensor parallelism against bf16: the 8B shapes of bench.py (d = 4096, 32 heads, 32 layers,
ff = 12288, L = 2414) sharded over tp in {2, 4, 8} ranks, both precisions timed alternately in one process.

On one GPU, per tp and per rank, timed with CUDA events (20 calls each after two warm-up calls):
  qkv / attn_out / gate_up / ff_out   the rank's four linear launches: QKV + RoPE + V^T, the attn_out GEMM pushing fp32 partial
                                      rows to the owners' receive buffers, gate/up + SwiGLU, the ff_out push; bf16 and FP8;
  quant_att / quant_h                 the local e4m3 quantiser the FP8 forward runs before attn_out / ff_out (1 x 128 groups);
  quant_xn                            the quantiser of the replicated activations [L, d] a rank would run before its QKV and
                                      gate/up GEMMs if the reduce broadcast bf16 (the work the fused FP8 reduce removes);
  reduce                              one rank's reduce + residual + norm + broadcast (rendezvous, reduce and wait launches),
                                      bf16 form and FP8 form, averaged over the tp ranks;
  sim_rank                            one forward of the 32 layers issued op by op for all tp simulated ranks on one stream (the
                                      sequence of mmdp_tp_forward), divided by tp; bf16 and FP8 alternately, two forwards each.
                                      Every layer reuses one layer's shard weights (the times depend on the shapes only). The ranks'
                                      NVLink traffic becomes local stores and every reduce call is preceded by the small fills that
                                      set the flags it waits on: a per-rank compute time, not the time of a real TP forward.
Under torchrun with >= 2 GPUs (tp = world size) it also times whole 512x512 samples of bench.py's workload through
generate_ti2ti with TensorParallelLLaDA in both precisions (--steps samples after --warmup, alternating); with one GPU those are
printed as "not measured". The GPU's name, power limit and SM clock are read in the same run. Prints one JSON line.

    python tools/bench_tp_fp8.py [--out FILE]
    torchrun --nproc-per-node 8 tools/bench_tp_fp8.py --steps 1 --warmup 0
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes as C
import io
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import CODEBOOK, GEN, MODEL_8B, TEXT_VOCAB, model_namespace, synthetic_layout  # noqa: E402
from tools.bench_gqa import gpu_info, time_op  # noqa: E402
from tools.bench_tp_gqa import synthetic_state_dict  # noqa: E402

L = 2414
TPS = (2, 4, 8)


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class Rank:
    """One simulated rank's layer shard in both precisions, its buffers and peer-visible state."""

    def __init__(self, tp, g, dev):
        from mmada_parallel_b200 import _lib
        d, ff, H = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["n_heads"]
        self.Hl = H // tp
        da, ffl = self.Hl * 128, ff // tp
        self.da, self.ffl = da, ffl

        def mk(*shape):
            return (torch.randn(*shape, device=dev, generator=g) * 0.02).to(torch.bfloat16)

        def q8(w):  # one scale per row over this slice (the times depend on the shapes only)
            q, s = _lib.quantize_fp8(w, w.shape[1])
            return q.view(torch.uint8), s[0].contiguous()

        self.wqkv, self.wo, self.w13, self.w2 = mk(3 * da, d), mk(d, da), mk(2 * ffl, d), mk(d, ffl)
        (self.wqkv8, self.sqkv), (self.wo8, self.so), (self.w13_8, self.s13), (self.w2_8, self.s2) = (
            q8(w) for w in (self.wqkv, self.wo, self.w13, self.w2))
        self.norm = torch.ones(d, dtype=torch.bfloat16, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.q, self.att, self.k = torch.empty(L, da, **bf), torch.empty(L, da, **bf), torch.empty(L, da, **bf)
        self.h = torch.empty(L, ffl, **bf)
        self.vt = torch.zeros(1, self.Hl, 128, (L + 7) // 8 * 8, **bf)
        R = (L + tp - 1) // tp
        self.xn = torch.zeros(L, d, **bf)
        self.xq = torch.zeros(L, d, dtype=torch.uint8, device=dev)
        self.xs = torch.ones(d // 128, L, dtype=torch.float32, device=dev)
        ka = max(da, ffl, d)
        self.a8 = torch.empty(L * ka, dtype=torch.uint8, device=dev)
        self.a8s = torch.empty(L * ka // 128, dtype=torch.float32, device=dev)
        self.x = torch.zeros(R, d, **bf)
        self.flags = torch.zeros(2, 8, dtype=torch.int32, device=dev)
        self.done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.recv = [torch.zeros(tp, R, d, dtype=torch.float32, device=dev) for _ in range(2)]

    def qkv(self, fp8, cos, sin, s):
        from mmada_parallel_b200._lib import check, lib
        d, Lpad = MODEL_8B["d_model"], self.vt.shape[-1]
        if fp8:
            check(lib.mmdp_qkv_rope_tp_fp8(self.xq.data_ptr(), d, self.xs.data_ptr(), self.wqkv8.data_ptr(), self.sqkv.data_ptr(), None, L, d,
                                           self.Hl, self.Hl, L, Lpad, cos.data_ptr(), sin.data_ptr(), self.q.data_ptr(), self.k.data_ptr(),
                                           self.vt.data_ptr(), s))
        else:
            check(lib.mmdp_qkv_rope_tp(self.xn.data_ptr(), d, self.wqkv.data_ptr(), L, d, self.Hl, L, Lpad, cos.data_ptr(), sin.data_ptr(),
                                       self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), s))

    def attention(self, s):
        from mmada_parallel_b200._lib import check, lib
        check(lib.mmdp_attention(self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), self.att.data_ptr(), 1, self.Hl, L,
                                 self.vt.shape[-1], 128 ** -0.5, s))

    def quant(self, x, K, s):
        from mmada_parallel_b200._lib import check, lib
        check(lib.mmdp_quantize_fp8(x.data_ptr(), K, L, K, 128, self.a8.data_ptr(), K, self.a8s.data_ptr(), s))

    def attn_out(self, fp8, recv_arr, tp, my, s):
        from mmada_parallel_b200._lib import check, lib
        d, da, R = MODEL_8B["d_model"], self.da, (L + tp - 1) // tp
        if fp8:
            self.quant(self.att, da, s)
            check(lib.mmdp_gemm_fp8_f32_scatter(self.a8.data_ptr(), da, self.a8s.data_ptr(), self.wo8.data_ptr(), da, self.so.data_ptr(), L, d,
                                                da, recv_arr, tp, R, my, s))
        else:
            check(lib.mmdp_gemm_f32_scatter(self.att.data_ptr(), da, self.wo.data_ptr(), da, L, d, da, recv_arr, tp, R, my, s))

    def gate_up(self, fp8, s):
        from mmada_parallel_b200._lib import EPI_SWIGLU, check, lib
        d, ffl = MODEL_8B["d_model"], self.ffl
        if fp8:
            check(lib.mmdp_gemm_fp8(EPI_SWIGLU, self.xq.data_ptr(), d, self.xs.data_ptr(), self.w13_8.data_ptr(), d, self.s13.data_ptr(), L,
                                    2 * ffl, d, self.h.data_ptr(), ffl, None, 0, s))
        else:
            check(lib.mmdp_gemm_bf16(EPI_SWIGLU, self.xn.data_ptr(), d, self.w13.data_ptr(), d, L, 2 * ffl, d, self.h.data_ptr(), ffl, None, 0, s))

    def ff_out(self, fp8, recv_arr, tp, my, s):
        from mmada_parallel_b200._lib import check, lib
        d, ffl, R = MODEL_8B["d_model"], self.ffl, (L + tp - 1) // tp
        if fp8:
            self.quant(self.h, ffl, s)
            check(lib.mmdp_gemm_fp8_f32_scatter(self.a8.data_ptr(), ffl, self.a8s.data_ptr(), self.w2_8.data_ptr(), ffl, self.s2.data_ptr(), L,
                                                d, ffl, recv_arr, tp, R, my, s))
        else:
            check(lib.mmdp_gemm_f32_scatter(self.h.data_ptr(), ffl, self.w2.data_ptr(), ffl, L, d, ffl, recv_arr, tp, R, my, s))


class Sim:
    def __init__(self, ranks):
        self.ranks, self.tp = ranks, len(ranks)
        self.xn_arr, self.fl_arr = _ptrs([rk.xn for rk in ranks]), _ptrs([rk.flags for rk in ranks])
        self.xq_arr, self.xs_arr = _ptrs([rk.xq for rk in ranks]), _ptrs([rk.xs for rk in ranks])
        self.recv_arr = [_ptrs([rk.recv[b] for rk in ranks]) for b in range(2)]

    def reduce_all(self, fp8, n_src, buf, ep, s):
        """Every rank's reduce call; before it, every flag it waits on already holds the call's epoch."""
        from mmada_parallel_b200._lib import check, lib
        d, tp = MODEL_8B["d_model"], self.tp
        R = (L + tp - 1) // tp
        for my, rk in enumerate(self.ranks):
            rk.flags.fill_(ep)
            r0 = my * R
            recv = rk.recv[buf].data_ptr() if n_src else None
            if fp8:
                check(lib.mmdp_tp_reduce_norm_fp8(recv, R, n_src, self.xq_arr, self.xs_arr, L, self.fl_arr, tp, my, rk.x.data_ptr(),
                                                  rk.norm.data_ptr(), r0, min(R, L - r0), d, 1e-5, ep & 0xFFFFFFFF, rk.done.data_ptr(), s))
            else:
                check(lib.mmdp_tp_reduce_norm(recv, R, n_src, self.xn_arr, self.fl_arr, tp, my, rk.x.data_ptr(), rk.norm.data_ptr(), r0,
                                              min(R, L - r0), d, 1e-5, ep & 0xFFFFFFFF, rk.done.data_ptr(), s))

    def forward(self, fp8, cos, sin, n_layers, epoch):
        """One forward of n_layers for every simulated rank in turn (tests/test_gpu_tp_fp8.py::sim_tp_forward_fp8's order; the last
        reduce broadcasts bf16 in both precisions). Returns the last epoch used."""
        from mmada_parallel_b200._lib import stream_ptr
        s, tp = stream_ptr(), self.tp
        epoch += 1
        self.reduce_all(fp8, 0, 0, epoch, s)
        for li in range(n_layers):
            for my, rk in enumerate(self.ranks):
                rk.qkv(fp8, cos, sin, s)
                rk.attention(s)
                rk.attn_out(fp8, self.recv_arr[0], tp, my, s)
            epoch += 1
            self.reduce_all(fp8, tp, 0, epoch, s)
            for my, rk in enumerate(self.ranks):
                rk.gate_up(fp8, s)
                rk.ff_out(fp8, self.recv_arr[1], tp, my, s)
            epoch += 1
            self.reduce_all(fp8 and li + 1 < n_layers, tp, 1, epoch, s)
        return epoch


def one_gpu(dev):
    from mmada_parallel_b200.model import rope_tables
    cos, sin = (t.to(dev) for t in rope_tables(128, 500000.0, L))
    g = torch.Generator(device=dev).manual_seed(0)
    results = []
    d = MODEL_8B["d_model"]
    for tp in TPS:
        ranks = [Rank(tp, g, dev) for _ in range(tp)]
        for rk in ranks:
            rk.xn.normal_(0.0, 1.0, generator=g)
            rk.x.normal_(0.0, 1.0, generator=g)
            rk.att.normal_(0.0, 1.0, generator=g)
            rk.h.normal_(0.0, 1.0, generator=g)
        sim, rk0 = Sim(ranks), ranks[0]
        epoch = [0]

        def reduce_once(fp8):
            epoch[0] += 1
            sim.reduce_all(fp8, tp, 0, epoch[0], None)

        sim.reduce_all(True, 0, 0, 1, None)  # valid e4m3 activations in every rank's buffer
        epoch[0] = 1
        r = {"tp": tp, "qkv_N": 3 * rk0.da, "ff_out_K": rk0.ffl}
        for prec, fp8 in (("bf16", False), ("fp8", True)):
            r[f"qkv_ms_{prec}"] = round(time_op(lambda: rk0.qkv(fp8, cos, sin, None)), 4)
            r[f"attn_out_ms_{prec}"] = round(time_op(lambda: rk0.attn_out(fp8, sim.recv_arr[0], tp, 0, None)), 4)
            r[f"gate_up_ms_{prec}"] = round(time_op(lambda: rk0.gate_up(fp8, None)), 4)
            r[f"ff_out_ms_{prec}"] = round(time_op(lambda: rk0.ff_out(fp8, sim.recv_arr[1], tp, 0, None)), 4)
            r[f"reduce_ms_{prec}"] = round(time_op(lambda: reduce_once(fp8), reps=10) / tp, 4)
        # the quantiser launches alone (the attn_out / ff_out FP8 times above include them)
        r["quant_att_ms"] = round(time_op(lambda: rk0.quant(rk0.att, rk0.da, None)), 4)
        r["quant_h_ms"] = round(time_op(lambda: rk0.quant(rk0.h, rk0.ffl, None)), 4)
        r["quant_xn_ms"] = round(time_op(lambda: rk0.quant(rk0.xn, d, None)), 4)
        epoch[0] = sim.forward(False, cos, sin, MODEL_8B["n_layers"], epoch[0])  # warm-up of both
        epoch[0] = sim.forward(True, cos, sin, MODEL_8B["n_layers"], epoch[0])
        t = {"bf16": [], "fp8": []}
        for _ in range(2):
            for prec, fp8 in (("bf16", False), ("fp8", True)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                epoch[0] = sim.forward(fp8, cos, sin, MODEL_8B["n_layers"], epoch[0])
                e1.record()
                torch.cuda.synchronize()
                t[prec].append(round(e0.elapsed_time(e1) / tp, 2))
        r["sim_rank_forward_ms_bf16"], r["sim_rank_forward_ms_fp8"] = t["bf16"], t["fp8"]
        print(json.dumps(r), file=sys.stderr, flush=True)
        results.append(r)
        del ranks, rk0, sim
        torch.cuda.empty_cache()
    return results


def multi_gpu_samples(args, rank, world, dev):
    """Whole 512x512 samples through generate_ti2ti on a TP = world model, bf16 and FP8 alternating."""
    import torch.distributed as dist
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    lay = synthetic_layout(seed=0)
    kw = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    cfg = model_namespace(MODEL_8B)
    sd = synthetic_state_dict(MODEL_8B["n_heads"], False, dev)
    models = {p: TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=MODEL_8B["max_sequence_length"], device=dev,
                                     text_vocab_size=TEXT_VOCAB, codebook_size=CODEBOOK, precision=p) for p in ("bf16", "fp8")}
    del sd
    torch.cuda.empty_cache()
    times = {"bf16": [], "fp8": []}
    for i in range(args.warmup + args.steps):
        for p, m in models.items():
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
                times[p].append(round(e0.elapsed_time(e1) / 1e3, 3))
    dist.barrier()
    return {"tp": world, "sample_s_bf16": times["bf16"], "sample_s_fp8": times["fp8"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1, help="timed samples per precision under torchrun with >= 2 GPUs")
    ap.add_argument("--warmup", type=int, default=0, help="untimed samples per precision first")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tp_fp8: needs a CUDA device (H100)")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}"
    torch.cuda.set_device(dev)
    line = {"gpu": gpu_info(), "L": L, "model": "8B synthetic (bench.py shapes), multi-head"}
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
