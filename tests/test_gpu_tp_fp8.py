"""The tensor-parallel forward with FP8 (e4m3) block linears on ONE GPU (helpers of test_gpu_tp_ops.py / test_gpu_fp8.py):

  mmdp_gemm_fp8_f32               fp64 restatement of the partial sw[n] sum_g sa[g][m] sum_k A W, inside the e4m3 accumulation
                                  bound; rounded to bf16 it is bitwise mmdp_gemm_fp8's plain output
  mmdp_gemm_fp8_f32_scatter       every row bitwise at recv[row // R][slot][row % R] (ragged M, a tile spanning two owners)
  mmdp_tp_reduce_norm_fp8         bytes and scales bitwise mmdp_quantize_fp8(group 128) of the bf16 reduce's rows, n_src = 0 and
                                  n; x_shard bitwise the bf16 reduce's; every rank's buffers identical
  mmdp_tp_forward (1 rank, FP8)   multi-head, 4 kv heads + bias, MQA against oracle.fp8_tp (the x1.5 rule of test_gpu_fp8.py);
                                  two row chunks bitwise one chunk
  TP = 2 / 4 / 8 op by op         the FP8 sequence of mmdp_tp_forward on simulated ranks: e4m3 activations bitwise identical on
                                  every rank after every reduce, ln_f(x) against the TP oracle
  TensorParallelLLaDA(fp8)        tp = 1: logits, generate_ti2ti in lock-step with the oracle loop; a bf16 model is unchanged
  TP = 2 on two GPUs              tests/_tp_fp8_worker.py (skipped below 2 GPUs)

The safety rule of test_gpu_tp_ops.py holds: simulated ranks run one after another on one stream and every flag a reduce call
waits on holds the call's epoch before it is issued; mmdp_tp_forward only runs with one rank."""
import contextlib
import ctypes as C
import io
import math
import os
import subprocess
import sys

import pytest
import torch

from helpers import ROOT, GpuBackedOracleModel, load_golden
from oracle import fp8, fp8_tp, llada_gqa
from oracle import generate as G
from test_gpu_fp8 import _assert_as_close_as_torch, _on_gpu_fp32, u8
from test_gpu_tp_ops import GUARD, SimRanks, _ptrs, _rand_bf16, _set_partials, _stream
from tp_ops_ref import bitwise_mismatch, is_sentinel, norm_inputs, scatter_expected, scatter_mismatch, sentinel_f32

pytestmark = pytest.mark.gpu

DEV = "cuda"
SCALE = 1.0 / math.sqrt(128.0)


def _lib():
    from mmada_parallel_b200 import _lib
    return _lib


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the FP8 fp32-partial GEMM and its scatter
# ---------------------------------------------------------------------------------------------------------------------------
def _operands(M, N, K, seed):
    L = _lib()
    g = torch.Generator().manual_seed(seed)
    a = _rand_bf16(g, M, K, scale=0.5)
    w = _rand_bf16(g, N, K, scale=K ** -0.5)
    qa, sa = L.quantize_fp8(a, 128)
    qw, sw = L.quantize_fp8(w, K)
    return qa, sa, qw, sw[0].contiguous()


def gemm_fp8_f32(qa, sa, qw, sw, ldc=None):
    L = _lib()
    M, K = qa.shape
    N = qw.shape[0]
    c = sentinel_f32(M, ldc or N, device=DEV)
    L.check(L.lib.mmdp_gemm_fp8_f32(qa.data_ptr(), K, sa.data_ptr(), qw.data_ptr(), K, sw.data_ptr(), M, N, K, c.data_ptr(), c.stride(0),
                                    _stream()))
    return c


def gemm_fp8_scatter(qa, sa, qw, sw, recv, R, slot):
    L = _lib()
    M, K = qa.shape
    L.check(L.lib.mmdp_gemm_fp8_f32_scatter(qa.data_ptr(), qa.stride(0), sa.data_ptr(), qw.data_ptr(), K, sw.data_ptr(), M, qw.shape[0], K,
                                            _ptrs(recv), len(recv), R, slot, _stream()))


@pytest.mark.parametrize("M,N,K,ldc", [(335, 264, 256, None), (1, 8, 128, None), (129, 520, 128, 528), (2414, 4096, 1536, None),
                                       (2414, 4096, 512, None)])
def test_gemm_fp8_f32_against_fp64(M, N, K, ldc):
    """|err| <= abssum (2^-12 + num_k 2^-23): the e4m3 tensor-core sum of one k-block keeps about 13 bits of its absolute-value
    sum (test_gpu_fp8.assert_ulp), the fp32 promotion one rounding per k-block. Mean error far inside (from 1024 elements on)."""
    qa, sa, qw, sw = _operands(M, N, K, M + N + K)
    c = gemm_fp8_f32(qa, sa, qw, sw, ldc)
    a64, w64 = qa.double().view(M, K // 128, 128), qw.double().view(N, K // 128, 128)
    ref = torch.zeros(M, N, dtype=torch.float64, device=DEV)
    abssum = torch.zeros_like(ref)
    for g in range(K // 128):
        ref += sa[g].double().unsqueeze(1) * (a64[:, g] @ w64[:, g].t())
        abssum += sa[g].double().abs().unsqueeze(1) * (a64[:, g].abs() @ w64[:, g].abs().t())
    ref *= sw.double()
    abssum *= sw.double().abs()
    got = c[:, :N].double()
    err = (got - ref).abs()
    bound = abssum * (2.0 ** -12 + (K // 128) * 2.0 ** -23)
    assert (err <= bound).all(), f"{int((err > bound).sum())} elements outside the bound, max err / bound {float((err / bound).max()):.3f}"
    if got.numel() >= 1024:
        assert err.mean().item() <= 0.05 * bound.mean().item()
    if ldc:
        assert is_sentinel(c[:, N:]), "columns past N of a row with ldc > N must stay untouched"
    plain = _lib().gemm_fp8(qa, sa, qw, sw)
    assert bitwise_mismatch(c[:, :N].to(torch.bfloat16), plain) == 0, "bf16(fp32 partial) must be the plain epilogue's output"
    assert bitwise_mismatch(c, gemm_fp8_f32(qa, sa, qw, sw, ldc)) == 0, "bitwise repeatable"


@pytest.mark.parametrize("M,N,K,n", [(335, 264, 256, 1), (335, 264, 256, 2), (335, 264, 256, 3), (335, 264, 256, 8),
                                     (2414, 1024, 512, 8), (300, 1024, 384, 4), (9, 1024, 128, 4), (1, 8, 128, 1)])
def test_gemm_fp8_f32_scatter(M, N, K, n):
    """M = 335 at n = 2: R = 168, the tile of rows 128 .. 255 spans two owners; n = 3: R = 112, tiles span up to three. M = 9 at
    n = 4: rank 3 owns no row and its buffer stays untouched. Values bitwise the un-scattered result."""
    qa, sa, qw, sw = _operands(M, N, K, M + n)
    R = (M + n - 1) // n
    ref = gemm_fp8_f32(qa, sa, qw, sw)
    for slot in range(n):
        recv = [sentinel_f32(n, R, N, device=DEV) for _ in range(n)]
        gemm_fp8_scatter(qa, sa, qw, sw, recv, R, slot)
        err = scatter_mismatch(recv, scatter_expected(ref, n, R, slot))
        assert err is None, f"M={M} n={n} slot={slot}: {err}"
    if M == 9:
        assert is_sentinel(recv[3])


def test_gemm_fp8_f32_scatter_rejects_bad_layouts():
    L = _lib()
    qa, sa, qw, sw = _operands(10, 16, 128, 0)
    recv = [sentinel_f32(2, 4, 16, device=DEV) for _ in range(2)]
    for R, slot in ((4, 0), (0, 0), (5, 2), (5, -1)):
        with pytest.raises(L.MmdpError):
            gemm_fp8_scatter(qa, sa, qw, sw, recv, R, slot)
    torch.cuda.synchronize()
    assert all(is_sentinel(t) for t in recv), "a rejected call launches nothing"


# ---------------------------------------------------------------------------------------------------------------------------
# 2. reduce + residual + norm + e4m3 broadcast
# ---------------------------------------------------------------------------------------------------------------------------
class SimRanksFp8(SimRanks):
    """SimRanks plus every rank's e4m3 activation buffer [M + GUARD, d] and its scales [d / 128][M] (filled with sentinels)."""

    def __init__(self, n, M, d, n_recv=1):
        super().__init__(n, M, d, n_recv)
        self.xq = [torch.full((M + GUARD, d), 0x5A, dtype=torch.uint8, device=DEV) for _ in range(n)]
        self.xs = [sentinel_f32(d // 128, M, device=DEV) for _ in range(n)]
        self._xq_arr, self._xs_arr = _ptrs(self.xq), _ptrs(self.xs)

    def reduce_fp8(self, my, n_src, w, eps, epoch, buf=0):
        """SimRanks.reduce for mmdp_tp_reduce_norm_fp8, under the same safety rule."""
        L = _lib()
        r0, nr = self.rows(my)
        self.flags[my].fill_(epoch)
        for q in range(self.n):
            if q != my:
                self.flags[q][:, my] = epoch - 1
        L.check(L.lib.mmdp_tp_reduce_norm_fp8(self.recv[buf][my].data_ptr() if n_src else None, self.R, n_src, self._xq_arr, self._xs_arr,
                                              self.M, self._flag_arr, self.n, my, self.x[my].data_ptr(), w.data_ptr(), r0, nr, self.d, eps,
                                              epoch & 0xFFFFFFFF, self.done[my].data_ptr(), _stream()))
        for q in range(self.n):
            if q != my:
                assert self.flags[q][:, my].tolist() == [epoch, epoch], f"rank {my}: flags in rank {q}'s array"
        assert int(self.done[my].item()) == 0

    def assert_xq_identical(self, what):
        for r in range(1, self.n):
            assert torch.equal(self.xq[r], self.xq[0]) and torch.equal(self.xs[r], self.xs[0]), f"{what}: rank {r}'s e4m3 buffers differ"


@pytest.mark.parametrize("n,M,d", [(1, 37, 256), (2, 75, 1024), (4, 130, 2048), (8, 2414, 4096), (2, 33, 5120), (8, 67, 8192)])
def test_tp_reduce_norm_fp8(n, M, d):
    """The FP8 form against the bf16 form on the same inputs: x_shard bitwise, the broadcast bitwise mmdp_quantize_fp8(group =
    128) of the bf16 rows, in every rank's buffers, guard rows untouched. n_src = 0 (after the embedding) and n_src = n."""
    L = _lib()
    eps = 1e-5
    g = torch.Generator().manual_seed(n * 1000 + d)
    w = (1 + 0.1 * torch.randn(d, generator=g)).to(torch.bfloat16).to(DEV)
    for n_src in (0, n):
        f8, b16 = SimRanksFp8(n, M, d), SimRanks(n, M, d)
        for my in range(n):
            _, nr = f8.rows(my)
            x = norm_inputs(nr, d, seed=my + d + n_src)[0].to(DEV) * 64
            f8.x[my][:nr] = x
            b16.x[my][:nr] = x
        _set_partials(f8, seed=n + d)
        for my in range(n):
            b16.recv[0][my].copy_(f8.recv[0][my])
        for my in range(n):
            f8.reduce_fp8(my, n_src, w, eps, epoch=3)
            b16.reduce(my, n_src, w, eps, epoch=3)
        for my in range(n):
            assert bitwise_mismatch(f8.x[my], b16.x[my]) == 0, f"rank {my}: x_shard differs from the bf16 reduce's"
        q, s = L.quantize_fp8(b16.xn[0][:M], 128)
        for r in range(n):
            assert torch.equal(f8.xq[r][:M], u8(q)), f"n_src={n_src} rank {r}: e4m3 bytes differ from mmdp_quantize_fp8"
            assert torch.equal(f8.xs[r], s), f"n_src={n_src} rank {r}: scales differ from mmdp_quantize_fp8"
            assert (f8.xq[r][M:] == 0x5A).all(), "guard rows of the e4m3 buffer"
        f8.assert_xq_identical(f"n_src={n_src}")


def test_tp_reduce_norm_fp8_rejects_bad_arguments():
    L = _lib()
    sim = SimRanksFp8(2, 16, 256)
    w = torch.ones(256, dtype=torch.bfloat16, device=DEV)
    for d, ld_s in ((200, 16), (256, 7)):  # d not a multiple of 128; a scale stride below the rows
        with pytest.raises(L.MmdpError):
            L.check(L.lib.mmdp_tp_reduce_norm_fp8(None, sim.R, 0, sim._xq_arr, sim._xs_arr, ld_s, sim._flag_arr, 2, 1, sim.x[1].data_ptr(),
                                                  w.data_ptr(), 8, 8, d, 1e-5, 1, sim.done[1].data_ptr(), _stream()))
    torch.cuda.synchronize()
    assert all((t == 0x5A).all() for t in sim.xq) and all(is_sentinel(t) for t in sim.xs)
    assert all(int(f.abs().sum()) == 0 for f in sim.flags), "a rejected call launches nothing"


# ---------------------------------------------------------------------------------------------------------------------------
# 3. the FP8 tensor-parallel body: one rank, two chunks, simulated ranks
# ---------------------------------------------------------------------------------------------------------------------------
TINY = dict(d_model=2048, n_heads=16, n_layers=2, mlp_hidden_size=4096, vocab_size=512, max_sequence_length=512)
CONFIGS = {"mha": dict(), "kv4_bias": dict(n_kv_heads=4, include_qkv_bias=True), "mqa": dict(multi_query_attention=True)}
_MODEL = {}


def _tiny(name):
    if name not in _MODEL:
        cfg = llada_gqa.make_config(**TINY, **CONFIGS[name])
        _MODEL[name] = (cfg, llada_gqa.make_weights(cfg, seed=79))
    return _MODEL[name]


def _quantize_rows(w):
    q, s = _lib().quantize_fp8(w.to(DEV).contiguous(), w.shape[1])
    return u8(q), s[0]


def _shard(name, rank, tp):
    """bf16 shard (norms, bias, embedding) + FP8 shard of the linears; kv heads of the rank."""
    key = ("shard", name, rank, tp)
    if key not in _MODEL:
        from mmada_parallel_b200.tensor_parallel import kv_shard, shard_state_dict, shard_state_dict_fp8
        cfg, sd = _tiny(name)
        Hkv = llada_gqa.kv_heads(cfg)
        sh = shard_state_dict(sd, cfg.n_layers, cfg.n_heads, rank, tp, 0, cfg.vocab_size, n_kv_heads=Hkv, qkv_bias=cfg.include_qkv_bias)
        w = {k: v.to(DEV).contiguous() for k, v in sh.items() if k.split(".")[-1] not in ("wqkv", "wo", "w13", "w2")}
        w.update(shard_state_dict_fp8(sd, cfg.n_layers, cfg.n_heads, rank, tp, _quantize_rows, n_kv_heads=Hkv))
        _MODEL[key] = (w, kv_shard(cfg.n_heads, Hkv, rank, tp)[1])
    return _MODEL[key]


def _ids(B, L):
    g = torch.Generator().manual_seed(B * 1000 + L + 2)
    return torch.randint(0, TINY["vocab_size"], (B, L), generator=g)


def _oracle(name, B, L, tp):
    """ln_f(x) of oracle.fp8_tp on the CPU and the same oracle code run by torch on the GPU (fp32 matmuls), [B*L, d] each."""
    key = ("oracle", name, B, L, tp)
    if key not in _MODEL:
        cfg, sd = _tiny(name)
        with torch.no_grad():
            cpu = fp8_tp.hidden_tp_fp8(_ids(B, L), sd, cfg, tp).reshape(B * L, -1)
            eager = _on_gpu_fp32(lambda: fp8_tp.hidden_tp_fp8(_ids(B, L).to(DEV), {k: v.to(DEV) for k, v in sd.items()}, cfg, tp))
        _MODEL[key] = (cpu, eager.reshape(B * L, -1).cpu())
    return _MODEL[key]


def _rope():
    from mmada_parallel_b200.model import rope_tables
    cos, sin = rope_tables(128, 500000.0, TINY["max_sequence_length"])
    return cos.to(DEV), sin.to(DEV)


def assert_vs_oracle(got, name, B, L, tp, what):
    want, eager = _oracle(name, B, L, tp)
    g, w_, e = got.float().cpu(), want.float(), eager.float()
    ulp = w_.abs().max().item() * 2.0 ** -8
    err, err_e = (g - w_).abs(), (e - w_).abs()
    print(f"[{what}] vs oracle.fp8_tp: max {err.max().item() / ulp:.2f} ulp, mean {err.mean().item() / ulp:.4f} | torch on the GPU: max "
          f"{err_e.max().item() / ulp:.2f}, mean {err_e.mean().item() / ulp:.4f}")
    _assert_as_close_as_torch(err, err_e, ulp, what)


def tp1_forward_fp8(name, B, L, n_chunks=1, chunk_rows0=0, epoch0=0):
    """mmdp_tp_forward with one rank in FP8 on fresh buffers. Returns (xn [M, d], epoch_out)."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    w, Hkv = _shard(name, 0, 1)
    d, H, nl, ff = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size
    M, Lpad = B * L, (L + 7) // 8 * 8
    bf = dict(dtype=torch.bfloat16, device=DEV)
    keep = []
    layers, layers8 = (L_.TpLayer * nl)(), (L_.TpLayerFp8 * nl)()
    for i in range(nl):
        p = f"blocks.{i}."
        for n in ("attn_norm", "ff_norm"):
            setattr(layers[i], n, w[p + n].data_ptr())
        if cfg.include_qkv_bias:
            layers[i].bqkv = w[p + "bqkv"].data_ptr()
        for n, k in (("wqkv", "wqkv8"), ("wo", "wo8"), ("w13", "w13_8"), ("w2", "w2_8"), ("sqkv", "sqkv"), ("so", "so"), ("s13", "s13"),
                     ("s2", "s2")):
            setattr(layers8[i], n, w[p + k].data_ptr())
    cos, sin = _rope()
    q, att = (torch.empty(M, d, **bf) for _ in range(2))
    k = torch.empty(M, Hkv * 128, **bf)
    h = torch.empty(M, ff, **bf)
    vt = torch.zeros(B, Hkv, 128, Lpad, **bf)
    xn = torch.full((M, d), float("nan"), **bf)
    xq = torch.empty(M * d, dtype=torch.uint8, device=DEV)
    xs = torch.empty(M * d // 128, dtype=torch.float32, device=DEV)
    a8 = torch.empty(M * ff, dtype=torch.uint8, device=DEV)
    a8s = torch.empty(M * ff // 128, dtype=torch.float32, device=DEV)
    arrs = [_ptrs([xn]), _ptrs([xq]), _ptrs([xs])]
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = d, H, ff, nl, 1, 0
    c.n_kv_heads_local = Hkv
    c.rms_eps = cfg.rms_norm_eps
    c.layers, c.layers_fp8 = layers, layers8
    c.precision = L_.PRECISION_FP8
    c.wte, c.ln_f, c.vocab = w["wte"].data_ptr(), w["ln_f"].data_ptr(), w["wte"].shape[0]
    c.cos_tab, c.sin_tab = cos.data_ptr(), sin.data_ptr()
    c.q, c.k, c.att, c.h, c.vt = q.data_ptr(), k.data_ptr(), att.data_ptr(), h.data_ptr(), vt.data_ptr()
    c.xn, c.xq, c.xq_scales = (C.cast(a, C.POINTER(C.c_void_p)) for a in arrs)
    c.a8, c.a8_scales = a8.data_ptr(), a8s.data_ptr()
    c.n_chunks, c.chunk_rows0 = n_chunks, chunk_rows0
    sizes = [M] if n_chunks == 1 else [chunk_rows0, M - chunk_rows0]
    for ci, rows in enumerate(sizes):
        st = dict(x=torch.empty(rows, d, **bf), recv=[torch.empty(1, rows, d, dtype=torch.float32, device=DEV) for _ in range(2)],
                  flags=torch.zeros(2, 8, dtype=torch.int32, device=DEV), done=torch.zeros(1, dtype=torch.int32, device=DEV))
        pa = [_ptrs([st["recv"][0]]), _ptrs([st["recv"][1]]), _ptrs([st["flags"]])]
        keep += [st, pa]
        c.chunk[ci].x_shard = st["x"].data_ptr()
        c.chunk[ci].recv[0] = C.cast(pa[0], C.POINTER(C.c_void_p))
        c.chunk[ci].recv[1] = C.cast(pa[1], C.POINTER(C.c_void_p))
        c.chunk[ci].flags = C.cast(pa[2], C.POINTER(C.c_void_p))
        c.chunk[ci].done_counter = st["done"].data_ptr()
    ids = _ids(B, L).to(DEV)
    out = C.c_uint32(0)
    L_.check(L_.lib.mmdp_tp_forward(C.byref(c), ids.data_ptr(), B, L, epoch0 & 0xFFFFFFFF, C.byref(out), _stream()))
    torch.cuda.synchronize()
    assert not vt[..., L:].any(), "V^T pad columns must stay zero"
    del keep
    return xn, int(out.value)


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("B,L", [(1, 301), (2, 150)])
def test_tp_forward_fp8_one_rank_vs_oracle(name, B, L):
    cfg, _ = _tiny(name)
    xn, ep = tp1_forward_fp8(name, B, L, epoch0=7)
    assert ep == 7 + 2 * cfg.n_layers + 1
    assert_vs_oracle(xn, name, B, L, 1, f"tp_forward fp8 {name} 1 rank B={B} L={L}")
    xn2, _ = tp1_forward_fp8(name, B, L, epoch0=2 ** 32 - 3)
    assert bitwise_mismatch(xn2, xn) == 0, "repeated forwards must be bitwise equal"


@pytest.mark.parametrize("name,chunk_rows0", [("kv4_bias", 100), ("kv4_bias", 150), ("mha", 220), ("mqa", 150)])
def test_tp_forward_fp8_two_chunks_bitwise(name, chunk_rows0):
    """The FP8 GEMM has no split-K tail and every quantised group is one row's, so two row chunks (each with its own scale block
    and a8 region) give the one-chunk result bit for bit."""
    one, _ = tp1_forward_fp8(name, 2, 150)
    two, _ = tp1_forward_fp8(name, 2, 150, n_chunks=2, chunk_rows0=chunk_rows0, epoch0=100)
    assert bitwise_mismatch(two, one) == 0, f"two chunks at {chunk_rows0} differ from one"


def sim_tp_forward_fp8(name, tp, B, L):
    """The FP8 per-layer sequence of mmdp_tp_forward (csrc/api.cu) issued from Python for every simulated rank in turn: e4m3
    broadcast after the embedding and after attn_out, FP8 QKV on it, att and h quantised locally before the FP8 scatter GEMMs,
    the last reduce (ln_f) in bf16. After every reduce round every rank's buffers must be bitwise identical. Returns rank 0's xn."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    d, H, nl, ff, eps = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size, cfg.rms_norm_eps
    Hl, ffl = H // tp, ff // tp
    da = Hl * 128
    M, Lpad = B * L, (L + 7) // 8 * 8
    sim = SimRanksFp8(tp, M, d, n_recv=2)
    shards = [_shard(name, r, tp) for r in range(tp)]
    ws, Hkv = [s[0] for s in shards], shards[0][1]
    bf = dict(dtype=torch.bfloat16, device=DEV)
    q, att = (torch.empty(M, da, **bf) for _ in range(2))
    k = torch.empty(M, Hkv * 128, **bf)
    h = torch.empty(M, ffl, **bf)
    vt = torch.zeros(B, Hkv, 128, Lpad, **bf)
    cos, sin = _rope()
    ids = _ids(B, L).to(DEV).view(-1)
    s = _stream()
    for r in range(tp):
        r0, nr = sim.rows(r)
        L_.check(L_.lib.mmdp_embed(ids[r0:].data_ptr(), ws[r]["wte"].data_ptr(), sim.x[r].data_ptr(), nr, d, ws[r]["wte"].shape[0], s))
    epoch = 1
    for r in range(tp):
        sim.reduce_fp8(r, 0, ws[r]["blocks.0.attn_norm"], eps, epoch)
    sim.assert_xq_identical("after the embedding's norm")
    for li in range(nl):
        p = f"blocks.{li}."
        for r in range(tp):
            w, b = ws[r], ws[r].get(p + "bqkv")
            L_.check(L_.lib.mmdp_qkv_rope_tp_fp8(sim.xq[r].data_ptr(), d, sim.xs[r].data_ptr(), w[p + "wqkv8"].data_ptr(), w[p + "sqkv"].data_ptr(),
                                                 None if b is None else b.data_ptr(), M, d, Hl, Hkv, L, Lpad, cos.data_ptr(), sin.data_ptr(),
                                                 q.data_ptr(), k.data_ptr(), vt.data_ptr(), s))
            L_.check(L_.lib.mmdp_attention_gqa(q.data_ptr(), k.data_ptr(), vt.data_ptr(), att.data_ptr(), B, None, Hl, Hkv, L, Lpad, SCALE, s))
            qa, sa = L_.quantize_fp8(att, 128)
            gemm_fp8_scatter(qa, sa, w[p + "wo8"], w[p + "so"], sim.recv[0], sim.R, r)
        epoch += 1
        for r in range(tp):
            sim.reduce_fp8(r, tp, ws[r][p + "ff_norm"], eps, epoch, buf=0)
        sim.assert_xq_identical(f"layer {li} after attn_out")
        for r in range(tp):
            w = ws[r]
            L_.check(L_.lib.mmdp_gemm_fp8(L_.EPI_SWIGLU, sim.xq[r].data_ptr(), d, sim.xs[r].data_ptr(), w[p + "w13_8"].data_ptr(), d,
                                          w[p + "s13"].data_ptr(), M, 2 * ffl, d, h.data_ptr(), ffl, None, 0, s))
            qh, sh = L_.quantize_fp8(h, 128)
            gemm_fp8_scatter(qh, sh, w[p + "w2_8"], w[p + "s2"], sim.recv[1], sim.R, r)
        epoch += 1
        last = li + 1 == nl
        for r in range(tp):
            if last:
                sim.reduce(r, tp, ws[r]["ln_f"], eps, epoch, buf=1)
            else:
                sim.reduce_fp8(r, tp, ws[r][f"blocks.{li + 1}.attn_norm"], eps, epoch, buf=1)
        if last:
            sim.assert_xn_identical("ln_f")
        else:
            sim.assert_xq_identical(f"layer {li} after ff_out")
    return sim.xn[0][:M]


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("tp,B,L", [(2, 2, 150), (4, 1, 301), (8, 1, 301)])
def test_tp_forward_fp8_simulated_ranks(name, tp, B, L):
    """TP = 2 / 4 / 8 on one GPU (4 kv heads at TP = 8 and MQA: replicated kv heads) against oracle.fp8_tp over the same tp."""
    got = sim_tp_forward_fp8(name, tp, B, L)
    assert_vs_oracle(got, name, B, L, tp, f"simulated fp8 {name} TP={tp} B={B} L={L}")


# ---------------------------------------------------------------------------------------------------------------------------
# 4. the public model, precision="fp8"
# ---------------------------------------------------------------------------------------------------------------------------
_TP = {}


def tp_fp8_model(meta, precision="fp8"):
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    from helpers import tiny_cfg_and_weights
    key = (meta["weight_seed"], precision)
    if key not in _TP:
        cfg, sd = tiny_cfg_and_weights(meta)
        _TP[key] = (TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=3, precision=precision), cfg, sd)
    return _TP[key]


def test_tp1_fp8_logits_vs_oracle():
    g = load_golden("forward_tiny.pt")
    model, cfg, sd = tp_fp8_model(g["meta"])
    assert model.precision == "fp8" and "blocks.0.wqkv" not in model.w
    lg = model(g["ids"]).logits
    with torch.no_grad():
        want = fp8.forward_logits_fp8(g["ids"], sd, cfg).float()[0]
        eager = _on_gpu_fp32(lambda: fp8.forward_logits_fp8(g["ids"].cuda(), {k: v.cuda() for k, v in sd.items()}, cfg)).float()[0].cpu()
    got = lg[0].float().cpu()
    ulp = want.abs().max().item() * 2.0 ** -8
    err, err_e = (got - want).abs(), (eager - want).abs()
    print(f"[tp=1 fp8] logits vs oracle.fp8: max {err.max().item() / ulp:.2f} ulp, mean {err.mean().item() / ulp:.4f} | torch on the GPU: "
          f"max {err_e.max().item() / ulp:.2f}, mean {err_e.mean().item() / ulp:.4f}")
    _assert_as_close_as_torch(err, err_e, ulp, "tp=1 fp8 logits")
    assert torch.equal(model(g["ids2"]).logits[0], lg[0]), "CFG batch rows are independent"


def test_tp1_fp8_generate_lockstep_with_oracle():
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    t = load_golden("trajectory_a_tiny.pt")
    model, _, _ = tp_fp8_model(t["meta"])
    lay = t["layout"]
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    for run in t["runs"][:2]:
        torch.manual_seed(run["global_seed"])
        img_o, txt_o = G.generate_ti2ti(GpuBackedOracleModel(model), lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                        stable_sort=True, **args, **run["kwargs"])
        torch.manual_seed(run["global_seed"])
        with contextlib.redirect_stdout(io.StringIO()):
            got = generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]), **args, **run["kwargs"])
        assert got == (img_o, txt_o), run["name"]


def test_bf16_tp_model_unchanged_by_fp8_tp_model():
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    from helpers import tiny_cfg_and_weights
    g = load_golden("forward_tiny.pt")
    cfg, sd = tiny_cfg_and_weights(g["meta"])
    b16 = TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=2)
    before = b16(g["ids2"]).logits.clone()
    m8 = TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=2, precision="fp8")
    lg8 = m8(g["ids2"]).logits
    assert torch.equal(before, b16(g["ids2"]).logits)
    assert not torch.equal(lg8, before), "the FP8 model computes its own (quantised) logits"
    del m8
    assert torch.equal(before, b16(g["ids2"]).logits)


def test_tensor_parallel_fp8_two_gpus():
    """TP = 2 FP8 (tests/_tp_fp8_worker.py) against tp_size = 1 FP8: logits within the bound, identical ids on both ranks."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29647", os.path.join(ROOT, "tests", "_tp_fp8_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    print(p.stdout[-3000:])
    assert p.returncode == 0, p.stderr[-3000:]
    assert "TP_FP8_CHECK_OK" in p.stdout
