"""Packed batches on the tensor-parallel model: the 8B shapes of bench.py (d = 4096, 32 heads, 32 layers, ff = 12288) sharded over
tp in {2, 4, 8} ranks, N in {1, 2, 4} requests of different prompt lengths around a 512x512 sample (L ~ 2414) and a 256x256 one
(L ~ 850).

On one GPU, per (tp, grid, N), per rank and per request, timed with CUDA events:
  packed      one forward of the 32 layers over the N sequences packed end to end (the sequence of mmdp_tp_forward_packed: packed
              QKV + RoPE, packed attention, attn_out pushed to the owners, reduce + residual + norm + broadcast, SwiGLU, ff_out
              pushed, reduce), issued op by op for all tp simulated ranks on one stream;
  sequential  the same N sequences as N single-sequence forwards (the sequence of mmdp_tp_forward);
  qkv / attn  rank 0's packed QKV launch (mmdp_qkv_rope_tp_packed) and packed attention launch (mmdp_attention_gqa with the
              lengths) against the N single-sequence launches, 20 calls each.
Every layer reuses one layer's shard weights (the times depend on the shapes only). The ranks' NVLink traffic becomes local
stores and every reduce call is preceded by the small fills that set the flags it waits on, so these are per-rank compute
times, not the times of a real TP forward. Under torchrun with >= 2 GPUs (tp = world size) it also times generate_ti2ti_batch
against sequential generate_ti2ti calls on TensorParallelLLaDA; with one GPU those are printed as "not measured". The GPU's
name, power limit and SM clock are read in the same run. Prints one JSON line.

    python tools/bench_tp_batch.py [--out FILE]
    torchrun --nproc-per-node 8 tools/bench_tp_batch.py --steps 1 --warmup 0
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
from tools.bench_tp_gqa import synthetic_state_dict  # noqa: E402

TPS, NS = (2, 4, 8), (1, 2, 4)
# prompts of different lengths around each grid's sequence length (bench.py's layout: L = 2414 at 512x512)
GRIDS = {"512x512": [2414, 2398, 2431, 2405], "256x256": [850, 838, 866, 845]}
SCALE = 1.0 / math.sqrt(128.0)


class Rank:
    """One simulated rank's layer shard (multi-head, 32 kv heads), buffers for Mmax rows and peer-visible state."""

    def __init__(self, tp, Mmax, n_max, Lmax, g, dev):
        d, ff, H = MODEL_8B["d_model"], MODEL_8B["mlp_hidden_size"], MODEL_8B["n_heads"]
        self.Hl = H // tp
        da, ffl = self.Hl * 128, ff // tp

        def mk(*shape):
            return (torch.randn(*shape, device=dev, generator=g) * 0.02).to(torch.bfloat16)

        self.wqkv, self.wo, self.w13, self.w2 = mk(3 * da, d), mk(d, da), mk(2 * ffl, d), mk(d, ffl)
        self.norm = torch.ones(d, dtype=torch.bfloat16, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.q, self.att, self.k = torch.empty(Mmax, da, **bf), torch.empty(Mmax, da, **bf), torch.empty(Mmax, da, **bf)
        self.h = torch.empty(Mmax, ffl, **bf)
        self.vt = torch.zeros(n_max * self.Hl * 128 * ((Lmax + 7) // 8 * 8), **bf)
        self.row_map = torch.empty(Mmax, 2, dtype=torch.int32, device=dev)
        R = (Mmax + tp - 1) // tp
        self.xn = torch.empty(Mmax, d, **bf).normal_(0.0, 1.0, generator=g)
        self.x = torch.empty(R, d, **bf).normal_(0.0, 1.0, generator=g)
        self.flags = torch.zeros(2, 8, dtype=torch.int32, device=dev)
        self.done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.recv = [torch.zeros(tp, R, d, dtype=torch.float32, device=dev) for _ in range(2)]

    def qkv_attention(self, lens, cos, sin, s):
        """Packed (several lengths) or equal-length (one) QKV + RoPE and attention over the first sum(lens) rows."""
        from mmada_parallel_b200._lib import PRECISION_BF16, check, lib
        d, M, Lpad = MODEL_8B["d_model"], sum(lens), (max(lens) + 7) // 8 * 8
        c_lens = (C.c_int32 * len(lens))(*lens)
        if len(lens) > 1:
            check(lib.mmdp_qkv_rope_tp_packed(PRECISION_BF16, self.xn.data_ptr(), d, None, self.wqkv.data_ptr(), None, None, d, self.Hl,
                                              self.Hl, len(lens), c_lens, Lpad, cos.data_ptr(), sin.data_ptr(), self.q.data_ptr(),
                                              self.k.data_ptr(), self.vt.data_ptr(), self.row_map.data_ptr(), s))
        else:
            check(lib.mmdp_qkv_rope_tp(self.xn.data_ptr(), d, self.wqkv.data_ptr(), M, d, self.Hl, M, Lpad, cos.data_ptr(), sin.data_ptr(),
                                       self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), s))
        self.attention(lens, s)

    def attention(self, lens, s):
        from mmada_parallel_b200._lib import check, lib
        Lpad = (max(lens) + 7) // 8 * 8
        if len(lens) > 1:
            check(lib.mmdp_attention_gqa(self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), self.att.data_ptr(), len(lens),
                                         (C.c_int32 * len(lens))(*lens), self.Hl, self.Hl, 0, Lpad, SCALE, s))
        else:
            check(lib.mmdp_attention(self.q.data_ptr(), self.k.data_ptr(), self.vt.data_ptr(), self.att.data_ptr(), 1, self.Hl, lens[0], Lpad,
                                     SCALE, s))


def sim_forward(ranks, lens, cos, sin, n_layers, epoch):
    """One forward of n_layers over the sequences `lens` (packed when there are several) issued for every simulated rank in turn
    (tests/test_gpu_tp_batch.py::sim_tp_forward). Before each reduce call every flag it waits on already holds the call's epoch.
    Returns the last epoch used."""
    from mmada_parallel_b200._lib import EPI_SWIGLU, check, lib, stream_ptr
    tp, d, s, M = len(ranks), MODEL_8B["d_model"], stream_ptr(), sum(lens)
    R = (M + tp - 1) // tp
    xn_arr = (C.c_void_p * tp)(*[rk.xn.data_ptr() for rk in ranks])
    fl_arr = (C.c_void_p * tp)(*[rk.flags.data_ptr() for rk in ranks])
    recv_arr = [(C.c_void_p * tp)(*[rk.recv[b].data_ptr() for rk in ranks]) for b in range(2)]

    def reduce_all(n_src, buf, ep):
        for my, rk in enumerate(ranks):
            rk.flags.fill_(ep)  # the call waits on its own flag array only
            r0 = my * R
            check(lib.mmdp_tp_reduce_norm(rk.recv[buf].data_ptr() if n_src else None, R, n_src, xn_arr, fl_arr, tp, my, rk.x.data_ptr(),
                                          rk.norm.data_ptr(), r0, min(R, M - r0), d, 1e-5, ep & 0xFFFFFFFF, rk.done.data_ptr(), s))

    epoch += 1
    reduce_all(0, 0, epoch)
    for _ in range(n_layers):
        for my, rk in enumerate(ranks):
            rk.qkv_attention(lens, cos, sin, s)
            da = rk.q.shape[1]
            check(lib.mmdp_gemm_f32_scatter(rk.att.data_ptr(), da, rk.wo.data_ptr(), da, M, d, da, recv_arr[0], tp, R, my, s))
        epoch += 1
        reduce_all(tp, 0, epoch)
        for my, rk in enumerate(ranks):
            ffl = rk.h.shape[1]
            check(lib.mmdp_gemm_bf16(EPI_SWIGLU, rk.xn.data_ptr(), d, rk.w13.data_ptr(), d, M, 2 * ffl, d, rk.h.data_ptr(), ffl, None, 0, s))
            check(lib.mmdp_gemm_f32_scatter(rk.h.data_ptr(), ffl, rk.w2.data_ptr(), ffl, M, d, ffl, recv_arr[1], tp, R, my, s))
        epoch += 1
        reduce_all(tp, 1, epoch)
    return epoch


def _time(fn, reps=2):
    fn()  # warm-up: every shape of the timed window
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def one_gpu(dev):
    from mmada_parallel_b200.model import rope_tables
    Lmax = max(max(v) for v in GRIDS.values())
    cos, sin = (t.to(dev) for t in rope_tables(128, 500000.0, Lmax))
    g = torch.Generator(device=dev).manual_seed(0)
    nl = MODEL_8B["n_layers"]
    results = []
    for tp in TPS:
        ranks = [Rank(tp, sum(GRIDS["512x512"][:max(NS)]), max(NS), Lmax, g, dev) for _ in range(tp)]
        ep = [0]

        def run(lens_list):
            for lens in lens_list:
                ep[0] = sim_forward(ranks, lens, cos, sin, nl, ep[0])

        for grid, all_lens in GRIDS.items():
            for n in NS:
                lens = all_lens[:n]
                t_packed = _time(lambda: run([lens]))
                t_seq = _time(lambda: run([[L] for L in lens]))
                rk0 = ranks[0]
                t_qkv_p = time_op(lambda: rk0.qkv_attention(lens, cos, sin, None)) if n > 1 else None
                t_attn_p = time_op(lambda: rk0.attention(lens, None)) if n > 1 else None
                t_qkv_s = sum(time_op(lambda: rk0.qkv_attention([L], cos, sin, None)) for L in lens)
                t_attn_s = sum(time_op(lambda: rk0.attention([L], None)) for L in lens)
                r = {"tp": tp, "grid": grid, "N": n, "lens": lens,
                     "packed_ms_per_rank_per_request": round(t_packed / tp / n, 3),
                     "sequential_ms_per_rank_per_request": round(t_seq / tp / n, 3),
                     "packed_speedup": round(t_seq / t_packed, 3)}
                if n > 1:
                    # qkv: QKV launch + attention launch together; attn: the attention launch alone (QKV = the difference)
                    r.update({"qkv_ms_packed": round(t_qkv_p - t_attn_p, 4), "qkv_ms_sequential": round(t_qkv_s - t_attn_s, 4),
                              "attn_ms_packed": round(t_attn_p, 4), "attn_ms_sequential": round(t_attn_s, 4)})
                print(json.dumps(r), file=sys.stderr, flush=True)
                results.append(r)
        del ranks
        torch.cuda.empty_cache()
    return results


def multi_gpu_batches(args, rank, world, dev):
    """generate_ti2ti_batch against sequential generate_ti2ti calls of N 512x512 requests on a TP = world model."""
    import torch.distributed as dist
    from mmada_parallel_b200.generators.batch import generate_ti2ti_batch
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    cfg = model_namespace(MODEL_8B)
    sd = synthetic_state_dict(MODEL_8B["n_heads"], False, dev)
    m = TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=MODEL_8B["max_sequence_length"], max_batch=max(NS), device=dev,
                            text_vocab_size=TEXT_VOCAB, codebook_size=CODEBOOK)
    del sd
    torch.cuda.empty_cache()
    out = []
    for n in NS:
        lays = [synthetic_layout(seed=i) for i in range(n)]
        reqs = [dict({k: lay[k] for k in ("input_ids", "text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text",
                                            "uncon_image")}, **GEN) for lay in lays]
        times = {}
        for mode in ("sequential", "batch"):
            ts = []
            for i in range(args.warmup + args.steps):
                rs = [dict(r, generator=torch.Generator(device=dev).manual_seed(42 + j)) for j, r in enumerate(reqs)]
                dist.barrier()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                with contextlib.redirect_stdout(io.StringIO()):
                    torch.manual_seed(5)
                    if mode == "batch":
                        generate_ti2ti_batch(m, rs)
                    else:
                        for r in rs:
                            generate_ti2ti(m, **r)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    ts.append(round(e0.elapsed_time(e1) / 1e3, 3))
            times[mode + "_s"] = ts
        out.append({"tp": world, "N": n, **times})
    dist.barrier()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1, help="timed runs per N under torchrun with >= 2 GPUs")
    ap.add_argument("--warmup", type=int, default=0, help="untimed runs per N first")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tp_batch: needs a CUDA device (H100)")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}"
    torch.cuda.set_device(dev)
    line = {"gpu": gpu_info(), "model": "8B synthetic (bench.py shapes), multi-head"}
    with torch.no_grad():
        if world >= 2:
            import torch.distributed as dist
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
            line["batches"] = multi_gpu_batches(args, rank, world, dev)
            dist.destroy_process_group()
            if rank != 0:
                return
        else:
            line["batches"] = "not measured (needs torchrun with >= 2 GPUs)"
            line["per_rank"] = one_gpu(dev)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
