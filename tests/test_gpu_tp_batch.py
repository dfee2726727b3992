"""Packed variable-length batches on the tensor-parallel model, on ONE GPU (helpers of test_gpu_tp_ops.py):

  mmdp_qkv_rope_tp_packed        bf16 and FP8, multi-head, 4 kv heads + bias and MQA shards: each sequence's q / k rows and V^T
                                 block bitwise those of the shard projection run on that sequence alone; V^T pad columns zero
  mmdp_tp_forward_packed (1 rank) bf16 and FP8, multi-head and grouped-query/bias: each sequence bitwise mmdp_tp_forward of that
                                 sequence alone, within the oracle bounds of the equal-length tests, the epoch advances by
                                 2 n_layers + 1, two row chunks (boundary inside a sequence and at one) bitwise one chunk
  TP = 2 / 4 / 8 op by op        the packed per-layer sequence on simulated ranks: every reduce leaves all xn buffers bitwise
                                 identical, each sequence bitwise the simulated single-sequence forward (ragged row ownership)
  TensorParallelLLaDA(tp=1)      forward_rows_packed against forward_rows per sequence, alternating with growing and shrinking
                                 lengths; generate_ti2ti_batch against sequential generate_ti2ti calls (bf16 and FP8)
  errors                         ValueError / NotImplementedError before anything is launched; native refusals of bad tables
  TP = 2 on two GPUs             tests/_tp_batch_worker.py (skipped below 2 GPUs)

Split-K tail and attention split tail are off where results are compared bit for bit: which tiles they touch depends on the
problem size. The safety rule of test_gpu_tp_ops.py holds: simulated ranks run one after another on one stream, every flag a
reduce call waits on holds the call's epoch before it is issued, and mmdp_tp_forward(_packed) only runs with one rank."""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch

from helpers import ROOT, load_golden
from oracle import fp8_tp, llada, llada_gqa
from test_gpu_batch import _assert_same, _layout, _run_both, splits_off
from test_gpu_fp8 import _assert_as_close_as_torch, _on_gpu_fp32
from test_gpu_tp_ops import SimRanks, _ptrs, _rand_bf16, _stream, gemm_scatter, ulp_errors
from tp_ops_ref import bitwise_mismatch, sentinel_bf16

pytestmark = pytest.mark.gpu

DEV = "cuda"
THETA = 500000.0
SCALE = 1.0 / math.sqrt(128.0)


def _lib():
    from mmada_parallel_b200 import _lib
    return _lib


def _offs(lens):
    return [sum(lens[:i]) for i in range(len(lens))]


def _c_lens(lens):
    return (C.c_int32 * len(lens))(*lens)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. mmdp_qkv_rope_tp_packed
# ---------------------------------------------------------------------------------------------------------------------------
SHARDS = {"mha": (8, 8, False), "kv4_bias": (16, 4, True), "mqa": (8, 1, False)}   # (Hl, Hkv_l, bias)


def _qkv_alone(prec, a, sa, w, sw, b, d, Hl, Hkv, L, cos, sin):
    """The equal-length shard projection of one sequence: mmdp_qkv_rope_tp / _gqa (bf16) or _fp8."""
    L_ = _lib()
    Lpad = (L + 7) // 8 * 8
    q = torch.empty(L, Hl * 128, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(L, Hkv * 128, dtype=torch.bfloat16, device=DEV)
    vt = torch.zeros(1, Hkv, 128, Lpad, dtype=torch.bfloat16, device=DEV)
    args = (cos.data_ptr(), sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), _stream())
    bp = None if b is None else b.data_ptr()
    if prec == "fp8":
        L_.check(L_.lib.mmdp_qkv_rope_tp_fp8(a.data_ptr(), d, sa.data_ptr(), w.data_ptr(), sw.data_ptr(), bp, L, d, Hl, Hkv, L, Lpad, *args))
    elif Hkv == Hl and b is None:
        L_.check(L_.lib.mmdp_qkv_rope_tp(a.data_ptr(), d, w.data_ptr(), L, d, Hl, L, Lpad, *args))
    else:
        L_.check(L_.lib.mmdp_qkv_rope_tp_gqa(a.data_ptr(), d, w.data_ptr(), bp, L, d, Hl, Hkv, L, Lpad, *args))
    return q, k, vt


@pytest.mark.parametrize("lens", [[301], [1, 150, 77], [200, 8, 129, 64, 3]])
@pytest.mark.parametrize("shard", list(SHARDS))
@pytest.mark.parametrize("prec", ["bf16", "fp8"])
def test_qkv_rope_tp_packed_bitwise(prec, shard, lens):
    from mmada_parallel_b200.model import rope_tables
    L_ = _lib()
    Hl, Hkv, bias = SHARDS[shard]
    d, M, n = 2048, sum(lens), len(lens)
    Lpad = (max(lens) + 7) // 8 * 8
    g = torch.Generator().manual_seed(Hl * 10 + Hkv + M)
    a = _rand_bf16(g, M, d)
    w = _rand_bf16(g, (Hl + 2 * Hkv) * 128, d, scale=d ** -0.5)
    b = _rand_bf16(g, (Hl + 2 * Hkv) * 128, scale=0.25) if bias else None
    cos, sin = (t.to(DEV) for t in rope_tables(128, THETA, max(lens)))
    qw = sw = None
    if prec == "fp8":
        qw, sw = L_.quantize_fp8(w, d)
        qw, sw = qw.view(torch.uint8), sw[0].contiguous()
    q = torch.empty(M, Hl * 128, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(M, Hkv * 128, dtype=torch.bfloat16, device=DEV)
    vt = torch.zeros(n, Hkv, 128, Lpad, dtype=torch.bfloat16, device=DEV)
    row_map = torch.empty(M, 2, dtype=torch.int32, device=DEV)
    with splits_off():
        if prec == "fp8":
            qa, sa = L_.quantize_fp8(a, 128)
            A, SA, W, SW, P = qa.view(torch.uint8).data_ptr(), sa.data_ptr(), qw.data_ptr(), sw.data_ptr(), L_.PRECISION_FP8
        else:
            A, SA, W, SW, P = a.data_ptr(), None, w.data_ptr(), None, L_.PRECISION_BF16
        L_.check(L_.lib.mmdp_qkv_rope_tp_packed(P, A, d, SA, W, SW, None if b is None else b.data_ptr(), d, Hl, Hkv, n, _c_lens(lens), Lpad,
                                                cos.data_ptr(), sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(),
                                                row_map.data_ptr(), _stream()))
        for i, (o, L) in enumerate(zip(_offs(lens), lens)):
            ai = a[o:o + L].contiguous()
            if prec == "fp8":
                qai, sai = L_.quantize_fp8(ai, 128)
                q1, k1, vt1 = _qkv_alone(prec, qai.view(torch.uint8), sai, qw, sw, b, d, Hl, Hkv, L, cos, sin)
            else:
                q1, k1, vt1 = _qkv_alone(prec, ai, None, w, None, b, d, Hl, Hkv, L, cos, sin)
            what = f"{prec} {shard} sequence {i} of {lens}"
            assert bitwise_mismatch(q[o:o + L], q1) == 0, f"{what}: q"
            assert bitwise_mismatch(k[o:o + L], k1) == 0, f"{what}: k"
            assert bitwise_mismatch(vt[i, ..., :L], vt1[0, ..., :L]) == 0, f"{what}: V^T"
            assert not vt[i, ..., L:].any(), f"{what}: V^T pad columns must stay zero"


def test_qkv_rope_tp_packed_rejects_bad_tables():
    L_ = _lib()
    t = torch.zeros(64, 2048, dtype=torch.bfloat16, device=DEV)
    rm = torch.empty(64, 2, dtype=torch.int32, device=DEV)
    p = t.data_ptr()

    def call(n, lens, Lpad=64, prec=L_.PRECISION_BF16, Hkv=8, row_map=rm.data_ptr()):
        return L_.lib.mmdp_qkv_rope_tp_packed(prec, p, 2048, None, p, None, None, 2048, 8, Hkv, n, _c_lens(lens) if lens else None, Lpad,
                                              p, p, p, p, p, row_map, _stream())
    L_.lib.mmdp_launch_count(1)
    for args, msg in [((0, [8]), b"sequences"), ((65, [1] * 65), b"sequences"), ((2, [8, 0]), b"length 0"), ((1, [72]), b"length 72"),
                      ((1, [8], 60), b"multiple of 8"), ((1, [8], 64, 7), b"precision"), ((1, [8], 64, L_.PRECISION_FP8), b"scales"),
                      ((1, [8], 64, L_.PRECISION_BF16, 3), b"must divide"), ((1, [8], 64, L_.PRECISION_BF16, 8, None), b"null")]:
        assert call(*args) == -1, args
        assert msg in L_.lib.mmdp_last_error(), (args, L_.lib.mmdp_last_error())
    assert L_.lib.mmdp_launch_count(0) == 0


# ---------------------------------------------------------------------------------------------------------------------------
# 2. mmdp_tp_forward_packed with one rank
# ---------------------------------------------------------------------------------------------------------------------------
TINY = dict(d_model=2048, n_heads=16, n_layers=2, mlp_hidden_size=4096, vocab_size=512, max_sequence_length=512)
CONFIGS = {"mha": dict(), "kv4_bias": dict(n_kv_heads=4, include_qkv_bias=True), "mqa": dict(multi_query_attention=True)}
_MODEL = {}


def _tiny(name):
    if name not in _MODEL:
        cfg = llada_gqa.make_config(**TINY, **CONFIGS[name])
        _MODEL[name] = (cfg, llada_gqa.make_weights(cfg, seed=81))
    return _MODEL[name]


def _quantize_rows(w):
    q, s = _lib().quantize_fp8(w.to(DEV).contiguous(), w.shape[1])
    return q.view(torch.uint8), s[0]


def _shard(name, prec, rank, tp):
    key = ("shard", name, prec, rank, tp)
    if key not in _MODEL:
        from mmada_parallel_b200.tensor_parallel import kv_shard, shard_state_dict, shard_state_dict_fp8
        cfg, sd = _tiny(name)
        Hkv = llada_gqa.kv_heads(cfg)
        sh = shard_state_dict(sd, cfg.n_layers, cfg.n_heads, rank, tp, 0, cfg.vocab_size, n_kv_heads=Hkv, qkv_bias=cfg.include_qkv_bias)
        w = {k: v.to(DEV).contiguous() for k, v in sh.items()}
        if prec == "fp8":
            w.update(shard_state_dict_fp8(sd, cfg.n_layers, cfg.n_heads, rank, tp, _quantize_rows, n_kv_heads=Hkv))
        _MODEL[key] = (w, kv_shard(cfg.n_heads, Hkv, rank, tp)[1])
    return _MODEL[key]


def _ids(lens, seed=3):
    g = torch.Generator().manual_seed(seed + sum(lens))
    return torch.randint(0, TINY["vocab_size"], (sum(lens),), generator=g)


def _rope():
    from mmada_parallel_b200.model import rope_tables
    cos, sin = rope_tables(128, THETA, TINY["max_sequence_length"])
    return cos.to(DEV), sin.to(DEV)


def tp1_forward(name, prec, ids, lens=None, L=None, n_chunks=1, chunk_rows0=0, epoch0=0):
    """One-rank mmdp_tp_forward_packed over the sequences `lens` of ids (lens None: mmdp_tp_forward of one sequence of L rows) on
    fresh buffers. Returns (xn [M, d], epoch_out)."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    w, Hkv = _shard(name, prec, 0, 1)
    d, H, nl, ff = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size
    M = sum(lens) if lens else L
    n_seg = len(lens) if lens else 1
    Lpad = ((max(lens) if lens else L) + 7) // 8 * 8
    bf = dict(dtype=torch.bfloat16, device=DEV)
    keep = []
    layers, layers8 = (L_.TpLayer * nl)(), (L_.TpLayerFp8 * nl)()
    for i in range(nl):
        p = f"blocks.{i}."
        for n in ("wqkv", "wo", "w13", "w2", "attn_norm", "ff_norm"):
            setattr(layers[i], n, w[p + n].data_ptr())
        if cfg.include_qkv_bias:
            layers[i].bqkv = w[p + "bqkv"].data_ptr()
        if prec == "fp8":
            for n, k in (("wqkv", "wqkv8"), ("wo", "wo8"), ("w13", "w13_8"), ("w2", "w2_8"), ("sqkv", "sqkv"), ("so", "so"), ("s13", "s13"),
                         ("s2", "s2")):
                setattr(layers8[i], n, w[p + k].data_ptr())
    cos, sin = _rope()
    q, att = (torch.empty(M, d, **bf) for _ in range(2))
    k = torch.empty(M, Hkv * 128, **bf)
    h = torch.empty(M, ff, **bf)
    vt = torch.zeros(n_seg, Hkv, 128, Lpad, **bf)
    xn = sentinel_bf16(M, d, device=DEV)
    xq = torch.empty(M * d, dtype=torch.uint8, device=DEV)
    xs = torch.empty(M * d // 128, dtype=torch.float32, device=DEV)
    a8 = torch.empty(M * ff, dtype=torch.uint8, device=DEV)
    a8s = torch.empty(M * ff // 128, dtype=torch.float32, device=DEV)
    row_map = torch.empty(M, 2, dtype=torch.int32, device=DEV)
    arrs = [_ptrs([xn]), _ptrs([xq]), _ptrs([xs])]
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = d, H, ff, nl, 1, 0
    c.n_kv_heads_local = Hkv
    c.rms_eps = cfg.rms_norm_eps
    c.layers = layers
    c.wte, c.ln_f, c.vocab = w["wte"].data_ptr(), w["ln_f"].data_ptr(), w["wte"].shape[0]
    c.cos_tab, c.sin_tab = cos.data_ptr(), sin.data_ptr()
    c.q, c.k, c.att, c.h, c.vt = q.data_ptr(), k.data_ptr(), att.data_ptr(), h.data_ptr(), vt.data_ptr()
    c.xn = C.cast(arrs[0], C.POINTER(C.c_void_p))
    if prec == "fp8":
        c.precision, c.layers_fp8 = L_.PRECISION_FP8, layers8
        c.xq, c.xq_scales = (C.cast(a, C.POINTER(C.c_void_p)) for a in arrs[1:])
        c.a8, c.a8_scales = a8.data_ptr(), a8s.data_ptr()
    c.packed.seg_pos, c.packed.max_rows, c.packed.rope_len = row_map.data_ptr(), M, TINY["max_sequence_length"]
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
    ids_d = ids.to(DEV)
    out = C.c_uint32(0)
    if lens:
        L_.check(L_.lib.mmdp_tp_forward_packed(C.byref(c), ids_d.data_ptr(), n_seg, _c_lens(lens), epoch0 & 0xFFFFFFFF, C.byref(out), _stream()))
    else:
        L_.check(L_.lib.mmdp_tp_forward(C.byref(c), ids_d.data_ptr(), 1, L, epoch0 & 0xFFFFFFFF, C.byref(out), _stream()))
    torch.cuda.synchronize()
    for i, Li in enumerate(lens or [L]):
        assert not vt[i, ..., Li:].any(), "V^T pad columns must stay zero"
    del keep
    return xn, int(out.value)


def _oracle(name, prec, ids):
    """ln_f(x) of one sequence by the CPU oracle (oracle.llada_gqa, or oracle.fp8_tp at tp = 1) and, for FP8, the same oracle code
    run by torch on the GPU."""
    cfg, sd = _tiny(name)
    with torch.no_grad():
        if prec == "fp8":
            cpu = fp8_tp.hidden_tp_fp8(ids[None], sd, cfg, 1)[0]
            eager = _on_gpu_fp32(lambda: fp8_tp.hidden_tp_fp8(ids[None].to(DEV), {k: v.to(DEV) for k, v in sd.items()}, cfg, 1))[0].cpu()
            return cpu, eager
        x = torch.nn.functional.embedding(ids[None], sd["model.transformer.wte.weight"])
        pos_sin, pos_cos = llada.rotary_tables(128, cfg.rope_theta, ids.numel())
        for i in range(cfg.n_layers):
            x = llada_gqa.block_forward(x, sd, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos)
        return llada.rms_norm(x, sd["model.transformer.ln_f.weight"], cfg.rms_norm_eps)[0], None


PACKED_LENS = [150, 37, 301, 8]


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("prec", ["bf16", "fp8"])
def test_tp_forward_packed_one_rank(prec, name):
    """Per sequence bitwise mmdp_tp_forward of the sequence alone (splits off); with default options within the equal-length
    tests' oracle bounds; the epoch advances by 2 n_layers + 1; a repeated call is bitwise equal."""
    cfg, _ = _tiny(name)
    lens = PACKED_LENS
    ids = _ids(lens)
    with splits_off():
        xn, ep = tp1_forward(name, prec, ids, lens, epoch0=7)
        assert ep == 7 + 2 * cfg.n_layers + 1
        for o, L in zip(_offs(lens), lens):
            alone, _ = tp1_forward(name, prec, ids[o:o + L], L=L)
            assert bitwise_mismatch(xn[o:o + L], alone) == 0, f"{prec} {name}: sequence of {L} rows differs from its own forward"
    xn, _ = tp1_forward(name, prec, ids, lens, epoch0=2 ** 32 - 3)
    xn2, _ = tp1_forward(name, prec, ids, lens, epoch0=11)
    assert bitwise_mismatch(xn2, xn) == 0, "repeated packed forwards must be bitwise equal"
    for o, L in zip(_offs(lens), lens):
        if L < 37:
            continue
        want, eager = _oracle(name, prec, ids[o:o + L])
        if prec == "fp8":
            g, w_ = xn[o:o + L].float().cpu(), want.float()
            ulp = w_.abs().max().item() * 2.0 ** -8
            _assert_as_close_as_torch((g - w_).abs(), (eager.float() - w_).abs(), ulp, f"fp8 {name} L={L}")
        else:
            mx, mean, _ = ulp_errors(xn[o:o + L], want)
            print(f"[tp_forward_packed {name} L={L}] vs oracle: max {mx:.2f} ulp, mean {mean:.4f} ulp")
            assert mx <= 4 and mean <= 0.5, (name, L, mx, mean)


@pytest.mark.parametrize("name,prec", [("kv4_bias", "bf16"), ("mha", "bf16"), ("mqa", "fp8"), ("kv4_bias", "fp8")])
def test_tp_forward_packed_two_chunks_bitwise(name, prec):
    """lens 150 | 37 | 301 | 8: chunk_rows0 = 187 lies at a sequence boundary, 250 and 100 inside a sequence."""
    ids = _ids(PACKED_LENS)
    with splits_off():
        one, _ = tp1_forward(name, prec, ids, PACKED_LENS)
        for r0 in (187, 250, 100):
            two, _ = tp1_forward(name, prec, ids, PACKED_LENS, n_chunks=2, chunk_rows0=r0, epoch0=100)
            assert bitwise_mismatch(two, one) == 0, f"{prec} {name}: two chunks at {r0} differ from one"


def test_tp_forward_packed_rejects_bad_tables():
    """Every refusal comes before any launch."""
    L_ = _lib()
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.n_layers, c.n_ranks, c.rank = 2048, 16, 1, 2, 0
    ids = torch.zeros(600, dtype=torch.int64, device=DEV)
    row_map = torch.empty(600, 2, dtype=torch.int32, device=DEV)
    out = C.c_uint32(0)

    def call(lens, n=None):
        return L_.lib.mmdp_tp_forward_packed(C.byref(c), ids.data_ptr(), len(lens) if n is None else n, _c_lens(lens) if lens else None,
                                             0, C.byref(out), _stream())
    L_.lib.mmdp_launch_count(1)
    assert call([8]) == -1 and b"no packed row map" in L_.lib.mmdp_last_error()
    c.packed.seg_pos, c.packed.max_rows, c.packed.rope_len = row_map.data_ptr(), 400, 300
    for lens, n, msg in [([], 0, b"sequences"), ([1] * 65, None, b"sequences"), ([8, 0], None, b"length 0"), ([301], None, b"length 301"),
                         ([300, 101], None, b"exceed the workspace"), ([1], None, b"at least one row")]:
        assert call(lens, n) == -1, lens
        assert msg in L_.lib.mmdp_last_error(), (lens, L_.lib.mmdp_last_error())
    c.n_chunks, c.chunk_rows0 = 2, 40
    assert call([20, 20]) == -1 and b"chunk_rows0" in L_.lib.mmdp_last_error()
    c.chunk_rows0 = 39
    assert call([20, 20]) == -1 and b"at least one row" in L_.lib.mmdp_last_error()   # chunk 1 holds 1 row for 2 ranks
    assert L_.lib.mmdp_launch_count(0) == 0


# ---------------------------------------------------------------------------------------------------------------------------
# 3. simulated ranks, op by op
# ---------------------------------------------------------------------------------------------------------------------------
def sim_tp_forward(name, tp, ids, lens, packed):
    """The bf16 per-layer sequence of mmdp_tp_forward(_packed) issued from Python for every simulated rank in turn. packed: the
    QKV projection is mmdp_qkv_rope_tp_packed and attention mmdp_attention_gqa with the lengths; otherwise lens is one sequence
    run through the equal-length calls. After every reduce round all xn buffers must be bitwise identical. Returns rank 0's xn."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    d, H, nl, ff, eps = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size, cfg.rms_norm_eps
    Hl, ffl = H // tp, ff // tp
    da = Hl * 128
    M, n = sum(lens), len(lens)
    Lpad = (max(lens) + 7) // 8 * 8
    sim = SimRanks(tp, M, d, n_recv=2)
    shards = [_shard(name, "bf16", r, tp) for r in range(tp)]
    ws, Hkv = [s[0] for s in shards], shards[0][1]
    bf = dict(dtype=torch.bfloat16, device=DEV)
    q, att = (torch.empty(M, da, **bf) for _ in range(2))
    k = torch.empty(M, Hkv * 128, **bf)
    h = torch.empty(M, ffl, **bf)
    vt = torch.zeros(n, Hkv, 128, Lpad, **bf)
    row_map = torch.empty(M, 2, dtype=torch.int32, device=DEV)
    cos, sin = _rope()
    ids = ids.to(DEV)
    s = _stream()
    for r in range(tp):
        r0, nr = sim.rows(r)
        assert nr >= 1
        L_.check(L_.lib.mmdp_embed(ids[r0:].data_ptr(), ws[r]["wte"].data_ptr(), sim.x[r].data_ptr(), nr, d, ws[r]["wte"].shape[0], s))
    epoch = 1
    for r in range(tp):
        sim.reduce(r, 0, ws[r]["blocks.0.attn_norm"], eps, epoch)
    sim.assert_xn_identical("after the embedding's norm")
    for li in range(nl):
        p = f"blocks.{li}."
        for r in range(tp):
            b = ws[r].get(p + "bqkv")
            bp = None if b is None else b.data_ptr()
            if packed:
                L_.check(L_.lib.mmdp_qkv_rope_tp_packed(L_.PRECISION_BF16, sim.xn[r].data_ptr(), d, None, ws[r][p + "wqkv"].data_ptr(), None, bp,
                                                        d, Hl, Hkv, n, _c_lens(lens), Lpad, cos.data_ptr(), sin.data_ptr(), q.data_ptr(),
                                                        k.data_ptr(), vt.data_ptr(), row_map.data_ptr(), s))
                L_.check(L_.lib.mmdp_attention_gqa(q.data_ptr(), k.data_ptr(), vt.data_ptr(), att.data_ptr(), n, _c_lens(lens), Hl, Hkv, 0,
                                                   Lpad, SCALE, s))
            else:
                L = lens[0]
                if Hkv == Hl and b is None:
                    L_.check(L_.lib.mmdp_qkv_rope_tp(sim.xn[r].data_ptr(), d, ws[r][p + "wqkv"].data_ptr(), M, d, Hl, L, Lpad, cos.data_ptr(),
                                                     sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), s))
                else:
                    L_.check(L_.lib.mmdp_qkv_rope_tp_gqa(sim.xn[r].data_ptr(), d, ws[r][p + "wqkv"].data_ptr(), bp, M, d, Hl, Hkv, L, Lpad,
                                                         cos.data_ptr(), sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), s))
                L_.check(L_.lib.mmdp_attention_gqa(q.data_ptr(), k.data_ptr(), vt.data_ptr(), att.data_ptr(), 1, None, Hl, Hkv, L, Lpad,
                                                   SCALE, s))
            gemm_scatter(att, ws[r][p + "wo"], sim.recv[0], sim.R, r)
        epoch += 1
        for r in range(tp):
            sim.reduce(r, tp, ws[r][p + "ff_norm"], eps, epoch, buf=0)
        sim.assert_xn_identical(f"layer {li} after attn_out")
        for r in range(tp):
            L_.check(L_.lib.mmdp_gemm_bf16(L_.EPI_SWIGLU, sim.xn[r].data_ptr(), d, ws[r][p + "w13"].data_ptr(), d, M, 2 * ffl, d,
                                           h.data_ptr(), ffl, None, 0, s))
            gemm_scatter(h, ws[r][p + "w2"], sim.recv[1], sim.R, r)
        epoch += 1
        nxt = f"blocks.{li + 1}.attn_norm" if li + 1 < nl else "ln_f"
        for r in range(tp):
            sim.reduce(r, tp, ws[r][nxt], eps, epoch, buf=1)
        sim.assert_xn_identical(f"layer {li} after ff_out")
    for i, L in enumerate(lens):
        assert not vt[i, ..., L:].any(), "V^T pad columns must stay zero"
    return sim.xn[0][:M].clone()


@pytest.mark.parametrize("name", ["mha", "kv4_bias", "mqa"])
@pytest.mark.parametrize("tp,lens", [(2, [100, 37, 150]), (4, [150, 37, 8, 120]), (8, [301, 40, 57])])
def test_tp_forward_packed_simulated_ranks(name, tp, lens):
    """Ragged ownership: at TP = 2 rank 0 owns all of the first two sequences and part of the third. The partial sums are added
    in rank order whatever the row owner, so each sequence is bitwise the simulated forward of that sequence alone."""
    ids = _ids(lens)
    with splits_off():
        got = sim_tp_forward(name, tp, ids, lens, packed=True)
        for o, L in zip(_offs(lens), lens):
            alone = sim_tp_forward(name, tp, ids[o:o + L], [L], packed=False)
            assert bitwise_mismatch(got[o:o + L], alone) == 0, f"TP={tp} {name}: sequence of {L} rows differs from its own forward"


# ---------------------------------------------------------------------------------------------------------------------------
# 4. TensorParallelLLaDA(tp_size = 1)
# ---------------------------------------------------------------------------------------------------------------------------
_TP = {}


def tp_model(precision, collective="nccl", chunks=1):
    """TensorParallelLLaDA with tp_size = 1. collective="p2p": the model's peer-memory path with one rank (mmdp_tp_forward and
    mmdp_tp_forward_packed through the Python glue of a real TP group): its peer buffers are set up in a one-process gloo group,
    which tp_size = 1 otherwise never does (it takes the NCCL formulation)."""
    import tempfile

    import torch.distributed as dist
    from helpers import tiny_cfg_and_weights
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    key = (precision, collective, chunks)
    if key not in _TP:
        meta = load_golden("trajectory_a_tiny.pt")["meta"]
        cfg, sd = tiny_cfg_and_weights(meta)
        m = TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=3, precision=precision, chunks=chunks)
        if collective == "p2p":
            with tempfile.TemporaryDirectory() as tmp:
                dist.init_process_group("gloo", store=dist.FileStore(os.path.join(tmp, "store"), 1), rank=0, world_size=1)
                try:
                    m.collective = "p2p"
                    m._init_peer_buffers(None)
                finally:
                    dist.destroy_process_group()
        _TP[key] = (m, cfg)
    return _TP[key]


MODES = [("nccl", 1), ("p2p", 1), ("p2p", 2)]


@pytest.mark.parametrize("collective,chunks", MODES)
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_tp1_forward_rows_packed_equals_forward_rows(precision, collective, chunks):
    """Packed and equal-length forwards alternate on one model with growing and shrinking lengths (the V^T pad rule, including a
    layout whose stride stays and whose blocks only grow, so the buffer is kept): every sequence's logits (text rows x V and image
    rows x the codebook window) equal its own forward_rows, bit for bit. On the peer-memory path the packed context points at the
    packed V^T buffer; with chunks=2 the 1200-row batch runs as two row chunks, its sequences alone as one."""
    model, cfg = tp_model(precision, collective, chunks)
    V, col0, nc = model.vocab_rows, model.vq_col0, model.vq_cols
    g = torch.Generator().manual_seed(5)
    with splits_off():
        for lens in ([120, 40, 250], [30], [300, 7], [8, 200, 64], [64, 200, 100], [64, 200, 8], [500, 300, 400]):
            if lens == [64, 200, 100]:  # same stride, every block at least as long as before: the pad columns are still zero
                assert model._pvt_Lpad == 200 and model._pvt_len[:3] == [8, 200, 64]
            seqs = [torch.randint(0, cfg.vocab_size, (L,), generator=g).to(DEV) for L in lens]
            rows = [torch.arange(0, L, 3, dtype=torch.int32, device=DEV) for L in lens]
            offs = _offs(lens)
            ra = torch.cat([r + o for r, o in zip(rows, offs)])
            la, lb = model.forward_rows_packed(torch.cat(seqs), lens, rows_a=ra, rows_b=ra, col0_b=col0, ncols_b=nc)
            assert la.shape == (ra.numel(), V) and lb.shape == (ra.numel(), nc)
            j = 0
            for x, r in zip(seqs, rows):
                a1, b1 = model.forward_rows(x[None], rows_a=r, rows_b=r, col0_b=col0, ncols_b=nc)
                assert torch.equal(la[j:j + r.numel()], a1) and torch.equal(lb[j:j + r.numel()], b1), (precision, lens, x.numel())
                j += r.numel()
            if collective == "p2p":
                assert model._pctx[0].vt == model._pvt.data_ptr(), "the packed context must point at the packed V^T buffer"


@pytest.mark.parametrize("collective,chunks", MODES)
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_tp1_generate_ti2ti_batch_equals_sequential(precision, collective, chunks):
    """Requests of different lengths, grids, steps and CFG: ids, text, per-step traces and every generator's state equal
    sequential generate_ti2ti calls on the same tensor-parallel model (splits off)."""
    t = load_golden("trajectory_a_tiny.pt")
    lay = t["layout"]
    kw = {r["name"]: dict(r["kwargs"]) for r in t["runs"]}
    model, _ = tp_model(precision, collective, chunks)
    reqs = [dict(_layout(lay, 0, 4, 4, 1), **dict(kw["greedy_cfgimg4"], text_steps=8, timesteps=4), _seed=42),
            dict(_layout(lay, 9, 3, 5, 2), **dict(kw["canonical_temp1"], text_steps=6, timesteps=3), _seed=43),
            dict(_layout(lay, -7, 5, 4, 3), **dict(kw["both_cfg_texttemp"], text_steps=10, timesteps=5), _seed=44),
            dict(_layout(lay, 23, 2, 6, 4), **dict(kw["no_cfg"], text_steps=5, timesteps=2), _seed=45)]
    with splits_off():
        seq, bat = _run_both(model, reqs)
    _assert_same(seq, bat)


# ---------------------------------------------------------------------------------------------------------------------------
# 5. errors
# ---------------------------------------------------------------------------------------------------------------------------
def test_tp_forward_rows_packed_errors():
    L_ = _lib()
    model, cfg = tp_model("bf16")
    z = lambda n: torch.zeros(n, dtype=torch.int64, device=DEV)  # noqa: E731
    L_.lib.mmdp_launch_count(1)
    for ids, lens in [(z(40), [10, 10, 10, 10]), (z(0), []), (z(600), [600]), (z(10), [10, 0]), (z(11), [5, 5])]:
        with pytest.raises(ValueError):
            model.forward_rows_packed(ids, lens)
    assert L_.lib.mmdp_launch_count(0) == 0
    with pytest.raises(NotImplementedError):
        model.forward_rows_packed(z(20), [10, 10], row_windows=[None, (0, 5)])


# ---------------------------------------------------------------------------------------------------------------------------
# 6. TP = 2 on two GPUs
# ---------------------------------------------------------------------------------------------------------------------------
def test_tensor_parallel_batch_two_gpus():
    """tests/_tp_batch_worker.py: p2p packed logits within 4 ulp of the tp_size = 1 packed logits; identical ids on both ranks
    from generate_ti2ti_batch."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29647", os.path.join(ROOT, "tests", "_tp_batch_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    print(p.stdout[-3000:])
    assert p.returncode == 0, p.stderr[-3000:]
    assert "TP_BATCH_CHECK_OK" in p.stdout
