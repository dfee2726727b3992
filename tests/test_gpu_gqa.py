"""Grouped-query / multi-query attention and the q/k/v bias on the H100: the attention kernels against an fp32 torch reference,
the QKV epilogue against torch, the tiny models against the real reference's fixture (forward_gqa_tiny.pt) and the oracle loop,
production-shape blocks against the CPU oracle, the FP8 context against oracle.fp8_gqa, and packed / windowed forwards against
per-sequence ones."""
import contextlib
import io
import math

import pytest
import torch

from helpers import GpuBackedOracleModel, load_golden
from oracle import generate as G
from oracle import llada, llada_gqa
from test_gpu_kernels import assert_attention_close, attn_version  # noqa: F401  (attn_version: the kernel-generation fixture)

pytestmark = pytest.mark.gpu

SCALE = 1.0 / math.sqrt(128.0)


@contextlib.contextmanager
def split_tail(on):
    from mmada_parallel_b200 import _lib
    _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", int(on)))
    try:
        yield
    finally:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))


@contextlib.contextmanager
def splits_off():
    from mmada_parallel_b200 import _lib
    _lib.lib.mmdp_set_gemm_splitk(0)
    _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 0))
    try:
        yield
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))


def _vt(v, lens, Hkv, Lpad):
    vt = torch.zeros(len(lens), Hkv, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    o = 0
    for i, L in enumerate(lens):
        vt[i, :, :, :L] = v[o:o + L].view(L, Hkv, 128).permute(1, 2, 0)
        o += L
    return vt


def _ref_attention(q, k, v, H, Hkv):
    L = q.shape[0]
    qh = q.view(L, H, 128).transpose(0, 1).float()
    kh = k.view(L, Hkv, 128).transpose(0, 1).float().repeat_interleave(H // Hkv, dim=0)
    vh = v.view(L, Hkv, 128).transpose(0, 1).float().repeat_interleave(H // Hkv, dim=0)
    return (torch.softmax(qh @ kh.transpose(-1, -2) * SCALE, dim=-1) @ vh).transpose(0, 1).reshape(L, H * 128)


# ---------------------------------------------------------------------------------------------------------------------
# 1. attention kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,Hkv", [(32, 8), (32, 1), (4, 2)])
@pytest.mark.parametrize("L", [1, 129, 2414])
def test_gqa_attention(H, Hkv, L, attn_version):
    from mmada_parallel_b200 import _lib
    torch.manual_seed(H * 1000 + Hkv * 10 + L)
    q = torch.randn(L, H * 128, device="cuda").to(torch.bfloat16)
    k = torch.randn(L, Hkv * 128, device="cuda").to(torch.bfloat16)
    v = torch.randn(L, Hkv * 128, device="cuda").to(torch.bfloat16)
    Lpad = (L + 7) // 8 * 8
    vt = _vt(v, [L], Hkv, Lpad)
    ref = _ref_attention(q, k, v, H, Hkv)
    for split in (1, 0):
        with split_tail(split):
            out = _lib.attention_gqa(q, k, vt, H, Hkv, SCALE, B=1, L=L)
        assert_attention_close(out, ref, f"gqa attention H={H} Hkv={Hkv} L={L} split_tail={split}")
    # the grouped kernel reads kv head h / G exactly as the multi-head kernel reads the repeated k / v
    G_ = H // Hkv
    k_rep = k.view(L, Hkv, 128).repeat_interleave(G_, dim=1).reshape(L, H * 128).contiguous()
    vt_rep = vt.repeat_interleave(G_, dim=1).contiguous()
    with split_tail(0):
        assert torch.equal(_lib.attention_gqa(q, k, vt, H, Hkv, SCALE, B=1, L=L), _lib.attention(q, k_rep, vt_rep, 1, H, L, SCALE))


@pytest.mark.parametrize("H,Hkv", [(32, 8), (32, 1), (4, 2)])
def test_gqa_attention_packed(H, Hkv, attn_version):
    from mmada_parallel_b200 import _lib
    lens = [1, 129, 700, 2414] if H == 32 else [1, 63, 129, 1000, 2414]
    M = sum(lens)
    Lpad = (max(lens) + 7) // 8 * 8
    torch.manual_seed(5 + H + Hkv)
    q = torch.randn(M, H * 128, device="cuda").to(torch.bfloat16)
    k = torch.randn(M, Hkv * 128, device="cuda").to(torch.bfloat16)
    v = torch.randn(M, Hkv * 128, device="cuda").to(torch.bfloat16)
    vt = _vt(v, lens, Hkv, Lpad)
    offs = [sum(lens[:i]) for i in range(len(lens))]
    out = {}
    for split in (1, 0):
        with split_tail(split):
            out[split] = _lib.attention_gqa(q, k, vt, H, Hkv, SCALE, seq_lens=lens)
    with split_tail(0):  # split tail off: each sequence equals its own launch bit for bit
        for i, (o, L) in enumerate(zip(offs, lens)):
            Lp = (L + 7) // 8 * 8
            alone = _lib.attention_gqa(q[o:o + L].contiguous(), k[o:o + L].contiguous(), vt[i:i + 1, :, :, :Lp].contiguous(), H, Hkv,
                                       SCALE, B=1, L=L)
            assert torch.equal(out[0][o:o + L], alone), (L, H, Hkv)
    for o, L in zip(offs, lens):
        ref = _ref_attention(q[o:o + L], k[o:o + L], v[o:o + L], H, Hkv)
        for split in (1, 0):
            assert_attention_close(out[split][o:o + L], ref, f"packed gqa attention L={L} H={H} Hkv={Hkv} split_tail={split}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. QKV epilogue: bias before the rounding, rotary on q and k heads, V^T per kv head (tiles that straddle k | v included)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,Hkv,L,bias", [(32, 1, 2414, True), (32, 8, 2414, True), (32, 8, 300, False), (4, 2, 129, True),
                                          (4, 1, 70, True)])
def test_qkv_epilogue_gqa(H, Hkv, L, bias):
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import rope_tables
    d, dkv = H * 128, Hkv * 128
    torch.manual_seed(H + Hkv + L)
    a = torch.randn(L, d, device="cuda").to(torch.bfloat16)
    w = (torch.randn(d + 2 * dkv, d, device="cuda") * d ** -0.5).to(torch.bfloat16)
    b = (torch.randn(d + 2 * dkv, device="cuda") * 0.25).to(torch.bfloat16) if bias else None
    cos, sin = rope_tables(128, 500000.0, L)
    cos, sin = cos.cuda(), sin.cuda()
    for mode in (2, 0):  # the split-K finishing pass (where the plan splits) and whole tiles
        _lib.lib.mmdp_set_gemm_splitk(mode)
        try:
            q, k, vt = _lib.qkv_rope_gqa(a, w, b, H, Hkv, L, cos, sin)
        finally:
            _lib.lib.mmdp_set_gemm_splitk(2)
        acc = a.float() @ w.float().t()
        if bias:
            acc = acc + b.float()
        y = acc.to(torch.bfloat16)  # nn.Linear: one rounding of acc + bias
        s, c = llada.rotary_tables(128, 500000.0, L)
        s, c = s.cuda(), c.cuda()
        qh = y[:, :d].view(1, L, H, 128).transpose(1, 2)
        kh = y[:, d:d + dkv].view(1, L, Hkv, 128).transpose(1, 2)
        q_ref = llada.apply_rotary(s, c, qh.float()).to(torch.bfloat16).transpose(1, 2).reshape(L, d)
        k_ref = llada.apply_rotary(s, c, kh.float()).to(torch.bfloat16).transpose(1, 2).reshape(L, dkv)
        v_ref = y[:, d + dkv:].view(L, Hkv, 128).permute(1, 2, 0)
        # the GEMM's fp32 sum order differs from torch's, so a projection may round one bf16 ulp apart and the rotary mixes two
        # of them: bound 4 bf16 ulp of max(|element|, the row's largest magnitude); a wrong head, region or bias is O(1) off
        for got, want, what in [(q, q_ref, "q"), (k, k_ref, "k"), (vt[0, :, :, :L].transpose(-1, -2), v_ref.transpose(-1, -2), "v^T")]:
            w_ = want.float()
            err = (got.float() - w_).abs()
            tol = 4 * 2.0 ** -8 * torch.maximum(w_.abs(), w_.abs().amax(-1, keepdim=True))
            assert (err <= tol).all(), (what, mode, float(err.max()))
            assert err.mean().item() < 0.05 * 2.0 ** -8 * w_.abs().mean().item() * 8, (what, mode, float(err.mean()))
        assert not vt[0, :, :, L:].any()


# ---------------------------------------------------------------------------------------------------------------------
# 3. tiny models against the real reference's fixture and the oracle loop
# ---------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def gqa_model(name, precision="bf16", max_batch=3):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    key = (name, precision, max_batch)
    if key not in _MODELS:
        g = load_golden("forward_gqa_tiny.pt")
        cfg = llada_gqa.make_config(**g["meta"]["common"], **g["configs"][name]["config"])
        sd = llada_gqa.make_weights(cfg, seed=g["meta"]["weight_seed"])
        m = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=max_batch, precision=precision)
        m.load_state_dict(sd)
        _MODELS[key] = (m, cfg, sd)
    return _MODELS[key]


NAMES = ["h4_kv2_bias", "h4_mqa", "h2_kv2_bias"]


@pytest.mark.parametrize("name", NAMES)
def test_tiny_gqa_logits_vs_reference_golden(name):
    g = load_golden("forward_gqa_tiny.pt")
    c = g["configs"][name]
    model, cfg, _ = gqa_model(name)
    assert model.n_kv_heads == llada_gqa.kv_heads(cfg)
    lg = model(g["ids"], infer=True, use_cache=False).logits
    want = c["logits_cols"].float()
    tol = 4 * want.abs().max().item() * 2.0 ** -8
    err = (lg[0].cpu()[:, g["cols"]].float() - want).abs().max().item()
    assert err <= tol, (name, err, tol)
    lg2 = model(g["ids2"], infer=True, use_cache=False).logits
    assert torch.equal(lg2[0], lg[0])
    assert (lg2.cpu()[:, :, g["cols"]].float() - c["logits2_cols"].float()).abs().max().item() <= tol


@pytest.mark.parametrize("name", NAMES)
def test_tiny_gqa_generate_lockstep_with_oracle(name):
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    g = load_golden("forward_gqa_tiny.pt")
    model, _, _ = gqa_model(name)
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


def test_tiny_gqa_refuses_token_cache():
    model, _, _ = gqa_model("h4_mqa")
    model.caching(True)
    try:
        with pytest.raises(NotImplementedError, match="token-cache"):
            model(torch.zeros(1, 16, dtype=torch.long), infer=True, use_cache=True)
    finally:
        model.caching(False)


# ---------------------------------------------------------------------------------------------------------------------
# 4. packed and windowed forwards equal per-sequence forwards (splits off), both precisions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
@pytest.mark.parametrize("name", ["h4_kv2_bias", "h4_mqa"])
def test_packed_and_windowed_equal_per_sequence(name, precision):
    model, cfg, _ = gqa_model(name, precision)
    V = cfg.vocab_size
    torch.manual_seed(11)
    lens = [70, 33, 129]
    seqs = [torch.randint(0, 126000, (L,), device="cuda") for L in lens]
    offs = [sum(lens[:i]) for i in range(len(lens))]
    with splits_off():
        rows = torch.cat([torch.arange(o, o + L, dtype=torch.int32, device="cuda") for o, L in zip(offs, lens)])
        packed, img = model.forward_rows_packed(torch.cat(seqs), lens, rows_a=rows, rows_b=rows, col0_b=126356, ncols_b=8192)
        for s, o, L in zip(seqs, offs, lens):
            r = torch.arange(L, dtype=torch.int32, device="cuda")
            alone, alone_b = model.forward_rows(s[None], rows_a=r, rows_b=r, col0_b=126356, ncols_b=8192)
            assert torch.equal(packed[o:o + L], alone) and torch.equal(img[o:o + L], alone_b), (name, precision, L)
            full = model(s[None], infer=True).logits[0]
            assert torch.equal(full, alone)
            # the last block's row window: rows inside it are unchanged
            lo, hi = L // 3, L // 3 + max(1, L // 4)
            rw = torch.arange(lo, hi, dtype=torch.int32, device="cuda")
            win, _ = model.forward_rows(s[None], rows_a=rw, row_window=(lo, hi))
            model.raise_device_errors()
            assert torch.equal(win, full[lo:hi]), (name, precision, L)
    assert packed.shape == (sum(lens), V)


# ---------------------------------------------------------------------------------------------------------------------
# 5. FP8 context against oracle.fp8_gqa
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_tiny_gqa_fp8_vs_fp8_oracle(name):
    from oracle import fp8_gqa
    from test_gpu_fp8 import _assert_as_close_as_torch, _on_gpu_fp32
    g = load_golden("forward_gqa_tiny.pt")
    model, cfg, sd = gqa_model(name, "fp8")
    lg = model(g["ids"], infer=True, use_cache=False).logits
    with torch.no_grad():
        want = fp8_gqa.forward_logits_fp8(g["ids"], sd, cfg).float()[0]
        eager = _on_gpu_fp32(lambda: fp8_gqa.forward_logits_fp8(g["ids"].cuda(), {k: v.cuda() for k, v in sd.items()}, cfg)).float()[0].cpu()
    got = lg[0].float().cpu()
    ulp = want.abs().max().item() * 2.0 ** -8
    err, err_e = (got - want).abs(), (eager - want).abs()
    print(f"[fp8 gqa {name}] max {err.max().item() / ulp:.2f} ulp, mean {err.mean().item() / ulp:.4f} | torch on the GPU: "
          f"max {err_e.max().item() / ulp:.2f}, mean {err_e.mean().item() / ulp:.4f}")
    _assert_as_close_as_torch(err, err_e, ulp, f"fp8 {name} logits")


# ---------------------------------------------------------------------------------------------------------------------
# 6. production shapes: one block + restricted head at d=4096, 32 heads, L=2414
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_kv_heads,mqa,bias", [(8, None, True), (None, True, False)])
def test_full_size_gqa_block_and_head_vs_oracle(n_kv_heads, mqa, bias):
    """As test_full_size_block_and_head_vs_oracle (test_gpu_model.py) for H=32 with 8 kv heads and a q/k/v bias (QKV N = 6144),
    and for multi-query attention (N = 4352: the k | v boundary at column 4224 lies inside a 256-wide tile): within 4 bf16 ulp
    of the tensor's scale of the CPU oracle, and a mean error at most 1.5x that of the same oracle run by torch on the GPU."""
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from test_gpu_model import _device_view_bf16
    cfg = llada_gqa.make_config(d_model=4096, n_heads=32, n_layers=1, mlp_hidden_size=12288, vocab_size=134656, max_sequence_length=2432,
                            n_kv_heads=n_kv_heads, multi_query_attention=mqa, include_qkv_bias=bias)
    g = torch.Generator(device="cuda").manual_seed(2025)
    d, ff, V, L = 4096, 12288, 134656, 2414
    dkv = llada_gqa.kv_heads(cfg) * 128

    def rnd(*s, std):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16)

    p = "model.transformer.blocks.0."
    sd = {"model.transformer.wte.weight": rnd(V, d, std=0.02), "model.transformer.ff_out.weight": rnd(V, d, std=d ** -0.5),
          "model.transformer.ln_f.weight": (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)}
    for n, shape, std in [("q_proj", (d, d), d ** -0.5), ("k_proj", (dkv, d), d ** -0.5), ("v_proj", (dkv, d), d ** -0.5),
                          ("attn_out", (d, d), d ** -0.5), ("ff_proj", (ff, d), d ** -0.5), ("up_proj", (ff, d), d ** -0.5),
                          ("ff_out", (d, ff), ff ** -0.5)]:
        sd[p + n + ".weight"] = rnd(*shape, std=std)
    if bias:
        for n, rows in [("q_proj", d), ("k_proj", dkv), ("v_proj", dkv)]:
            sd[p + n + ".bias"] = rnd(rows, std=0.25)
    sd[p + "attn_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)
    sd[p + "ff_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=2432, max_batch=1)
    m.load_state_dict(sd)
    ids = torch.randint(0, 126000, (1, L), device="cuda", generator=g)
    text_rows = torch.arange(2157, 2413, dtype=torch.int32, device="cuda")
    img_rows = torch.arange(1100, 1100 + 1024, dtype=torch.int32, device="cuda")
    a, b = m.forward_rows(ids, rows_a=text_rows, rows_b=img_rows, col0_b=126356, ncols_b=8192)
    hidden = _device_view_bf16(_lib.lib.mmdp_model_hidden(m._h), L * d).view(L, d).clone()
    torch.cuda.synchronize()
    del m

    def oracle(w, ids_, dev):
        with torch.no_grad():
            x = torch.nn.functional.embedding(ids_, w["model.transformer.wte.weight"])
            pos_sin, pos_cos = llada.rotary_tables(128, cfg.rope_theta, L)
            x = llada_gqa.block_forward(x, w, p, cfg, pos_sin.to(dev), pos_cos.to(dev))
            xn = llada.rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)[0]
            head = w["model.transformer.ff_out.weight"]
            return (x[0], torch.nn.functional.linear(xn[2157:2413], head),
                    torch.nn.functional.linear(xn[1100:1100 + 1024], head[126356:126356 + 8192]))

    want = oracle({k: v.cpu() for k, v in sd.items()}, ids.cpu(), "cpu")
    eager = oracle(sd, ids, "cuda")
    failures = []
    for got, e, w, what in zip((hidden, a, b), eager, want, ("residual stream", "text-row logits", "image-row codebook logits")):
        gq, eq, wq = got.float().cpu(), e.float().cpu(), w.float()
        ulp = wq.abs().max().item() * 2.0 ** -8
        err, err_e = (gq - wq).abs(), (eq - wq).abs()
        print(f"[full-size gqa kv={llada_gqa.kv_heads(cfg)} bias={bias}] {what}: native max {err.max().item() / ulp:.2f} ulp, mean "
              f"{err.mean().item() / ulp:.4f} | torch eager max {err_e.max().item() / ulp:.2f}, mean {err_e.mean().item() / ulp:.4f}")
        if not torch.isfinite(gq).all():
            failures.append((what, "non-finite"))
        if err.max().item() > 4 * ulp:
            failures.append((what, "max", err.max().item() / ulp))
        if err.mean().item() > 1.5 * err_e.mean().item() + 0.02 * ulp:
            failures.append((what, "mean vs eager", err.mean().item() / ulp, err_e.mean().item() / ulp))
    assert not failures, failures
