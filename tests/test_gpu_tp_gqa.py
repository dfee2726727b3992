"""Tensor-parallel grouped-query / multi-query attention and the q/k/v bias on ONE GPU (helpers of test_gpu_tp_ops.py):

  mmdp_qkv_rope_tp_gqa          every rank's q / k / V^T bitwise equal to its slice of mmdp_qkv_rope_gqa on the full weight
                                (split-K off) and inside the fp32-reference bounds of test_qkv_epilogue_gqa; V^T pad columns zero
  mmdp_tp_forward (1 rank)      a d = 2048, H = 16 model with 4 kv heads + bias and with MQA, within 4 bf16 ulp of oracle.llada_gqa
  TP = 2 / 4 / 8 op by op       the grouped-query per-layer sequence of mmdp_tp_forward on simulated ranks (kv heads replicated
                                at Hkv = 4, TP = 8): every reduce leaves all xn buffers bitwise identical
  two row chunks                bitwise equal to one chunk (the grouped-query epilogue with row0)
  TensorParallelLLaDA(tp=1)     the reference fixture's grouped-query configs: logits and the generation loop
  TP = 2 on two GPUs            tests/_tp_gqa_worker.py (skipped below 2 GPUs)

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
from oracle import generate as G
from oracle import llada, llada_gqa
from test_gpu_tp_ops import SimRanks, _Options, _ptrs, _rand_bf16, _stream, gemm_scatter, ulp_errors
from tp_ops_ref import bits, bitwise_mismatch, sentinel_bf16

pytestmark = pytest.mark.gpu

DEV = "cuda"
THETA = 500000.0
SCALE = 1.0 / math.sqrt(128.0)


def _lib():
    from mmada_parallel_b200 import _lib
    return _lib


# ---------------------------------------------------------------------------------------------------------------------------
# 1. QKV + RoPE of a grouped-query shard
# ---------------------------------------------------------------------------------------------------------------------------
def qkv_rope_tp_gqa(a, wsh, bsh, d, Hl, Hkv_l, B, L, cos, sin):
    L_ = _lib()
    M, Lpad = B * L, (L + 7) // 8 * 8
    q = torch.empty(M, Hl * 128, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(M, Hkv_l * 128, dtype=torch.bfloat16, device=DEV)
    vt = torch.zeros(B, Hkv_l, 128, Lpad, dtype=torch.bfloat16, device=DEV)
    L_.check(L_.lib.mmdp_qkv_rope_tp_gqa(a.data_ptr(), a.stride(0), wsh.data_ptr(), None if bsh is None else bsh.data_ptr(), M, d, Hl,
                                         Hkv_l, L, Lpad, cos.data_ptr(), sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(),
                                         _stream()))
    return q, k, vt


def assert_qkv_vs_fp32(q, k, vt, a, wsh, bsh, Hl, Hkv_l, B, L, what):
    """The bounds of test_qkv_epilogue_gqa (test_gpu_gqa.py): nn.Linear rounds acc + bias once, rotary in fp32 on the rounded
    values; 4 bf16 ulp of max(|element|, the row's largest magnitude), mean far inside."""
    M, da, dkv = B * L, Hl * 128, Hkv_l * 128
    acc = a.float() @ wsh.float().t()
    if bsh is not None:
        acc = acc + bsh.float()
    y = acc.to(torch.bfloat16)
    s, c = llada.rotary_tables(128, THETA, L)
    s, c = s.to(DEV), c.to(DEV)
    qh = y[:, :da].view(B, L, Hl, 128).transpose(1, 2)
    kh = y[:, da:da + dkv].view(B, L, Hkv_l, 128).transpose(1, 2)
    q_ref = llada.apply_rotary(s, c, qh.float()).to(torch.bfloat16).transpose(1, 2).reshape(M, da)
    k_ref = llada.apply_rotary(s, c, kh.float()).to(torch.bfloat16).transpose(1, 2).reshape(M, dkv)
    v_ref = y[:, da + dkv:].view(B, L, Hkv_l, 128).permute(0, 2, 3, 1)            # [B, Hkv_l, 128, L]
    for got, want, name in [(q, q_ref, "q"), (k, k_ref, "k"), (vt[..., :L].transpose(-1, -2), v_ref.transpose(-1, -2), "v^T")]:
        w_ = want.float()
        err = (got.float() - w_).abs()
        tol = 4 * 2.0 ** -8 * torch.maximum(w_.abs(), w_.abs().amax(-1, keepdim=True))
        assert (err <= tol).all(), (what, name, float(err.max()))
        assert err.mean().item() < 0.05 * 2.0 ** -8 * w_.abs().mean().item() * 8, (what, name, float(err.mean()))
    assert not vt[..., L:].any(), f"{what}: V^T pad columns must stay zero"


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("H,Hkv,tp", [(32, 8, 2), (32, 8, 8), (32, 1, 4), (16, 4, 8)])
def test_qkv_rope_tp_gqa_shard(H, Hkv, tp, bias, B):
    """Every rank of the shard layout of tensor_parallel.shard_state_dict: (32, 8, 8) and (16, 4, 8) replicate each kv head on
    2 ranks, (32, 1, 4) is MQA; (16, 4, 8) has a 256-wide tile that holds the shard's k head and v head."""
    from mmada_parallel_b200.model import rope_tables
    from mmada_parallel_b200.tensor_parallel import kv_shard
    L = 201  # Lpad = 208: the V^T pad columns exist and must stay zero
    d, dkv, M = H * 128, Hkv * 128, B * L
    Hl, da = H // tp, (H // tp) * 128
    g = torch.Generator().manual_seed(H * 100 + Hkv * 10 + tp + B)
    a = _rand_bf16(g, M, d)
    wq = _rand_bf16(g, d, d, scale=d ** -0.5)
    wk, wv = (_rand_bf16(g, dkv, d, scale=d ** -0.5) for _ in range(2))
    bq, bk, bv = (_rand_bf16(g, n, scale=0.25) for n in (d, dkv, dkv)) if bias else (None, None, None)
    cos, sin = (t.to(DEV) for t in rope_tables(128, THETA, L))
    with _Options(splitk=0):
        q_full, k_full, vt_full = _lib().qkv_rope_gqa(a, torch.cat([wq, wk, wv]), torch.cat([bq, bk, bv]) if bias else None, H, Hkv,
                                                       L, cos, sin)
        for r in range(tp):
            kv0, n_kv = kv_shard(H, Hkv, r, tp)
            sl, kv = slice(r * da, (r + 1) * da), slice(kv0 * 128, (kv0 + n_kv) * 128)
            wsh = torch.cat([wq[sl], wk[kv], wv[kv]]).contiguous()
            bsh = torch.cat([bq[sl], bk[kv], bv[kv]]).contiguous() if bias else None
            q, k, vt = qkv_rope_tp_gqa(a, wsh, bsh, d, Hl, n_kv, B, L, cos, sin)
            assert_qkv_vs_fp32(q, k, vt, a, wsh, bsh, Hl, n_kv, B, L, f"rank {r} of {tp}")
            assert bitwise_mismatch(q, q_full[:, sl]) == 0, f"rank {r}: q differs from the full projection's heads"
            assert bitwise_mismatch(k, k_full[:, kv]) == 0, f"rank {r}: k differs from the full projection's kv heads"
            assert bitwise_mismatch(vt, vt_full[:, kv0:kv0 + n_kv]) == 0, f"rank {r}: V^T differs"


# ---------------------------------------------------------------------------------------------------------------------------
# 2. the tensor-parallel body: one rank, simulated ranks, two chunks
# ---------------------------------------------------------------------------------------------------------------------------
TINY = dict(d_model=2048, n_heads=16, n_layers=2, mlp_hidden_size=4096, vocab_size=512, max_sequence_length=512)
CONFIGS = {"kv4_bias": dict(n_kv_heads=4, include_qkv_bias=True), "mqa": dict(multi_query_attention=True)}
_MODEL = {}


def _tiny(name):
    if name not in _MODEL:
        cfg = llada_gqa.make_config(**TINY, **CONFIGS[name])
        _MODEL[name] = (cfg, llada_gqa.make_weights(cfg, seed=78))
    return _MODEL[name]


def _shard(name, rank, tp):
    key = ("shard", name, rank, tp)
    if key not in _MODEL:
        from mmada_parallel_b200.tensor_parallel import kv_shard, shard_state_dict
        cfg, sd = _tiny(name)
        Hkv = llada_gqa.kv_heads(cfg)
        sh = shard_state_dict(sd, cfg.n_layers, cfg.n_heads, rank, tp, 0, cfg.vocab_size, n_kv_heads=Hkv, qkv_bias=cfg.include_qkv_bias)
        w = {k: v.to(DEV).contiguous() for k, v in sh.items()}
        _MODEL[key] = (w, kv_shard(cfg.n_heads, Hkv, rank, tp)[1])
    return _MODEL[key]


def _ids(B, L):
    g = torch.Generator().manual_seed(B * 1000 + L + 1)
    return torch.randint(0, TINY["vocab_size"], (B, L), generator=g)


def _oracle_hidden(name, B, L):
    key = ("oracle", name, B, L)
    if key not in _MODEL:
        cfg, sd = _tiny(name)
        with torch.no_grad():
            x = torch.nn.functional.embedding(_ids(B, L), sd["model.transformer.wte.weight"])
            pos_sin, pos_cos = llada.rotary_tables(128, cfg.rope_theta, L)
            for i in range(cfg.n_layers):
                x = llada_gqa.block_forward(x, sd, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos)
            _MODEL[key] = llada.rms_norm(x, sd["model.transformer.ln_f.weight"], cfg.rms_norm_eps).reshape(B * L, -1)
    return _MODEL[key]


def _rope():
    from mmada_parallel_b200.model import rope_tables
    cos, sin = rope_tables(128, THETA, TINY["max_sequence_length"])
    return cos.to(DEV), sin.to(DEV)


def tp1_forward_gqa(name, B, L, n_chunks=1, chunk_rows0=0, epoch0=0):
    """test_gpu_tp_ops.tp1_forward for a grouped-query / biased shard: k [M, 128 Hkv_l], vt [B, Hkv_l, 128, Lpad], the layers'
    bqkv and the context's n_kv_heads_local. Returns (xn [M, d], epoch_out)."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    w, Hkv = _shard(name, 0, 1)
    d, H, nl, ff = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size
    M, Lpad = B * L, (L + 7) // 8 * 8
    bf = dict(dtype=torch.bfloat16, device=DEV)
    keep = []
    layers = (L_.TpLayer * nl)()
    for i in range(nl):
        p = f"blocks.{i}."
        for n in ("wqkv", "wo", "w13", "w2", "attn_norm", "ff_norm"):
            setattr(layers[i], n, w[p + n].data_ptr())
        if cfg.include_qkv_bias:
            layers[i].bqkv = w[p + "bqkv"].data_ptr()
    cos, sin = _rope()
    q, att = (torch.empty(M, d, **bf) for _ in range(2))
    k = torch.empty(M, Hkv * 128, **bf)
    h = torch.empty(M, ff, **bf)
    vt = torch.zeros(B, Hkv, 128, Lpad, **bf)
    xn = sentinel_bf16(M, d, device=DEV)
    xn_arr = _ptrs([xn])
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = d, H, ff, nl, 1, 0
    c.n_kv_heads_local = Hkv
    c.rms_eps = cfg.rms_norm_eps
    c.layers = layers
    c.wte, c.ln_f, c.vocab = w["wte"].data_ptr(), w["ln_f"].data_ptr(), w["wte"].shape[0]
    c.cos_tab, c.sin_tab = cos.data_ptr(), sin.data_ptr()
    c.q, c.k, c.att, c.h, c.vt = q.data_ptr(), k.data_ptr(), att.data_ptr(), h.data_ptr(), vt.data_ptr()
    c.xn = C.cast(xn_arr, C.POINTER(C.c_void_p))
    c.n_chunks, c.chunk_rows0 = n_chunks, chunk_rows0
    sizes = [M] if n_chunks == 1 else [chunk_rows0, M - chunk_rows0]
    for ci, rows in enumerate(sizes):
        st = dict(x=torch.empty(rows, d, **bf), recv=[torch.empty(1, rows, d, dtype=torch.float32, device=DEV) for _ in range(2)],
                  flags=torch.zeros(2, 8, dtype=torch.int32, device=DEV), done=torch.zeros(1, dtype=torch.int32, device=DEV))
        arrs = [_ptrs([st["recv"][0]]), _ptrs([st["recv"][1]]), _ptrs([st["flags"]])]
        keep += [st, arrs]
        c.chunk[ci].x_shard = st["x"].data_ptr()
        c.chunk[ci].recv[0] = C.cast(arrs[0], C.POINTER(C.c_void_p))
        c.chunk[ci].recv[1] = C.cast(arrs[1], C.POINTER(C.c_void_p))
        c.chunk[ci].flags = C.cast(arrs[2], C.POINTER(C.c_void_p))
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
def test_tp_forward_gqa_one_rank_vs_oracle(name, B, L):
    """ln_f(x) of every row within 4 bf16 ulp of the tensor's scale of oracle.llada_gqa, mean below half an ulp (the bounds of
    test_tp_forward_one_rank_vs_oracle); repeated calls bitwise equal."""
    cfg, _ = _tiny(name)
    xn, ep = tp1_forward_gqa(name, B, L, epoch0=7)
    assert ep == 7 + 2 * cfg.n_layers + 1
    mx, mean, _ = ulp_errors(xn, _oracle_hidden(name, B, L))
    print(f"[tp_forward gqa {name} 1 rank B={B} L={L}] vs oracle: max {mx:.2f} ulp, mean {mean:.4f} ulp")
    assert mx <= 4 and mean <= 0.5, (mx, mean)
    xn2, _ = tp1_forward_gqa(name, B, L, epoch0=2 ** 32 - 3)
    assert bitwise_mismatch(xn2, xn) == 0, "repeated forwards must be bitwise equal"


@pytest.mark.parametrize("chunk_rows0", [100, 150, 220])
def test_tp_forward_gqa_two_chunks_bitwise(chunk_rows0):
    """B = 2, L = 150, 4 kv heads and a bias: the chunk boundary inside batch row 0, at the batch boundary, inside batch row 1.
    The second chunk's grouped-query epilogue runs with row0 = chunk_rows0 (positions and V^T absolute, q / k relative to the
    chunk); split-K off, so every GEMM element has the same K order in both schedules."""
    with _Options(splitk=0):
        one, _ = tp1_forward_gqa("kv4_bias", 2, 150)
        two, _ = tp1_forward_gqa("kv4_bias", 2, 150, n_chunks=2, chunk_rows0=chunk_rows0, epoch0=100)
    diff = bits(two) != bits(one)
    assert not diff.any(), f"two chunks at {chunk_rows0}: {int(diff.sum())} elements differ (first row {int(diff.nonzero()[0, 0])})"


def sim_tp_forward_gqa(name, tp, B, L):
    """test_gpu_tp_ops.sim_tp_forward with the grouped-query shard: mmdp_qkv_rope_tp_gqa (with the shard's bias) and
    mmdp_attention_gqa on Hl query heads and Hkv_l kv heads, as mmdp_tp_forward issues them for such a shard. After every reduce
    round all xn buffers must be bitwise identical. Returns rank 0's xn."""
    L_ = _lib()
    cfg, _ = _tiny(name)
    d, H, nl, ff, eps = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size, cfg.rms_norm_eps
    Hl, ffl = H // tp, ff // tp
    da = Hl * 128
    M, Lpad = B * L, (L + 7) // 8 * 8
    sim = SimRanks(tp, M, d, n_recv=2)
    shards = [_shard(name, r, tp) for r in range(tp)]
    ws = [s[0] for s in shards]
    Hkv = shards[0][1]
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
            L_.check(L_.lib.mmdp_qkv_rope_tp_gqa(sim.xn[r].data_ptr(), d, ws[r][p + "wqkv"].data_ptr(), None if b is None else b.data_ptr(),
                                                 M, d, Hl, Hkv, L, Lpad, cos.data_ptr(), sin.data_ptr(), q.data_ptr(), k.data_ptr(),
                                                 vt.data_ptr(), s))
            L_.check(L_.lib.mmdp_attention_gqa(q.data_ptr(), k.data_ptr(), vt.data_ptr(), att.data_ptr(), B, None, Hl, Hkv, L, Lpad,
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
    return sim.xn[0][:M]


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("tp,B,L", [(2, 2, 150), (4, 1, 301), (8, 1, 301), (8, 2, 150)])
def test_tp_forward_gqa_simulated_ranks(name, tp, B, L):
    """TP = 2 / 4 / 8 on one GPU; with 4 kv heads at TP = 8 each kv head is computed on two ranks. Bounds of
    test_tp_forward_simulated_ranks: against the one-rank forward 4 ulp, mean 0.35 ulp; against the oracle 5 ulp, mean 0.5 ulp,
    at most 1 in 10^5 elements beyond 4 ulp."""
    got = sim_tp_forward_gqa(name, tp, B, L)
    one, _ = tp1_forward_gqa(name, B, L)
    mx1, mean1, _ = ulp_errors(got, one)
    mxo, meano, beyond = ulp_errors(got, _oracle_hidden(name, B, L))
    print(f"[simulated gqa {name} TP={tp} B={B} L={L}] vs one rank: max {mx1:.2f} ulp, mean {mean1:.4f} ulp | vs oracle: max "
          f"{mxo:.2f} ulp, mean {meano:.4f} ulp, beyond 4 ulp {beyond * got.numel():.0f} elements")
    assert mx1 <= 4 and mean1 <= 0.35, f"from the one-rank forward: max {mx1:.2f}, mean {mean1:.3f} ulp"
    assert mxo <= 5 and meano <= 0.5, f"from the oracle: max {mxo:.2f}, mean {meano:.3f} ulp"
    assert beyond <= 1e-5, f"from the oracle: {beyond * got.numel():.0f} elements beyond 4 ulp"


def test_tp_forward_rejects_bad_kv_heads():
    """n_kv_heads_local must divide n_heads_local; the call is refused before anything is launched."""
    L_ = _lib()
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.n_layers, c.n_ranks, c.n_kv_heads_local = 2048, 16, 1, 1, 3
    ids = torch.zeros(8, dtype=torch.int64, device=DEV)
    out = C.c_uint32(0)
    assert L_.lib.mmdp_tp_forward(C.byref(c), ids.data_ptr(), 1, 8, 0, C.byref(out), _stream()) == -1
    assert b"n_kv_heads_local=3" in L_.lib.mmdp_last_error()


# ---------------------------------------------------------------------------------------------------------------------------
# 3. the public tensor-parallel model on the reference fixture's grouped-query configs
# ---------------------------------------------------------------------------------------------------------------------------
NAMES = ["h4_kv2_bias", "h4_mqa", "h2_kv2_bias"]
_TP_MODELS = {}


def tp_gqa_model(name):
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    if name not in _TP_MODELS:
        g = load_golden("forward_gqa_tiny.pt")
        cfg = llada_gqa.make_config(**g["meta"]["common"], **g["configs"][name]["config"])
        sd = llada_gqa.make_weights(cfg, seed=g["meta"]["weight_seed"])
        _TP_MODELS[name] = TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=3)
    return _TP_MODELS[name]


@pytest.mark.parametrize("name", NAMES)
def test_tp1_gqa_logits_vs_reference_golden(name):
    """The bound of test_tiny_gqa_logits_vs_reference_golden: 4 bf16 ulp of the fixture's logits scale."""
    g = load_golden("forward_gqa_tiny.pt")
    c = g["configs"][name]
    model = tp_gqa_model(name)
    assert model.gqa
    lg = model(g["ids"]).logits
    want = c["logits_cols"].float()
    tol = 4 * want.abs().max().item() * 2.0 ** -8
    err = (lg[0].cpu()[:, g["cols"]].float() - want).abs().max().item()
    print(f"[tp=1 {name}] logits vs reference fixture: max {err / (tol / 4):.2f} ulp")
    assert err <= tol, (name, err, tol)
    lg2 = model(g["ids2"]).logits
    assert torch.equal(lg2[0], lg[0])
    assert (lg2.cpu()[:, :, g["cols"]].float() - c["logits2_cols"].float()).abs().max().item() <= tol


@pytest.mark.parametrize("name", NAMES)
def test_tp1_gqa_generate_lockstep_with_oracle(name):
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    g = load_golden("forward_gqa_tiny.pt")
    model = tp_gqa_model(name)
    lay = g["layout"]
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    for kw, seed in [(g["meta"]["greedy"], 42), (dict(g["meta"]["greedy"], temperature=1.0, text_temperature=0.7, cfg_scale=1.5), 7)]:
        torch.manual_seed(999)
        with contextlib.redirect_stdout(io.StringIO()):
            img, txt = generate_ti2ti(model, g["ids"], generator=torch.Generator().manual_seed(seed), **args, **kw)
        torch.manual_seed(999)
        img_o, txt_o = G.generate_ti2ti(GpuBackedOracleModel(model), g["ids"], generator=torch.Generator().manual_seed(seed),
                                        stable_sort=True, **args, **kw)
        assert img == img_o and txt == txt_o, (name, seed)


def test_tensor_parallel_gqa_two_gpus():
    """h4_kv2_bias and h4_mqa at TP = 2 (tests/_tp_gqa_worker.py): peer-memory logits within 4 ulp of the single-GPU model and of
    the NCCL collective, bitwise repeatable, the same ids on both ranks over a short generation."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29643", os.path.join(ROOT, "tests", "_tp_gqa_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    print(p.stdout[-3000:])
    assert p.returncode == 0, p.stderr[-3000:]
    assert "TP_GQA_CHECK_OK" in p.stdout
