"""wgmma GEMM / attention / norm kernels against fp32 torch references of the same op (floating-point kernels).
Tolerances: the outputs are bf16 roundings of fp32-accumulated results; a different accumulation order may move a value
across one rounding boundary, so the bound is 1 bf16 ulp of the result magnitude per bf16 rounding point on the path
(2 for the residual epilogue, 3 for SwiGLU), stated per test."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def bf(x):
    return x.to(torch.bfloat16)


def ref_linear(a, w):
    return bf(a.float() @ w.float().t())


def assert_ulp(got, want, ulps, what, mag=None):
    """|got - want| <= ulps * (bf16 spacing at the magnitude of the quantities that were rounded). `mag` carries the
    magnitude of the operands when the result is a sum that can cancel (residual add, rotary)."""
    g, w = got.float(), want.float()
    assert not torch.isnan(g).any(), what
    scale = w.abs().max().clamp_min(1e-20)
    ref_mag = w.abs() if mag is None else torch.maximum(w.abs(), mag.float().abs())
    # bf16 spacing at magnitude m is <= m * 2^-7; tiny entries are bounded by the spacing at 1/64 of the max
    tol = ulps * torch.maximum(ref_mag, scale / 64) * 2.0 ** -7
    bad = (g - w).abs() > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} outside {ulps} ulp; max abs err {float((g - w).abs().max())}"
    assert (g != w).float().mean() < 0.02, f"{what}: too many roundings differ"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (1, 8, 8), (333, 264, 200), (512, 1024, 1024), (2414, 4096, 512), (77, 8192, 256)])
def test_gemm_plain(M, N, K):
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M + N + K)
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    assert_ulp(_lib.gemm_bf16(a, w), ref_linear(a, w), 1, f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("M", [5900, 7242])
def test_gemm_grouped_tile_order(M):
    """More than 45 m-tiles switch the persistent GEMM to the grouped-M tile order (gemm.cu / gemm_tile_coords): plain and
    residual epilogues (the latter with its split-K tail) against the fp32 reference, and bit-identical to the plain order."""
    import os
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M)
    K, N = 512, 1024
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    r = bf(torch.randn(M, N, device="cuda"))
    lin = ref_linear(a, w)
    got = _lib.gemm_bf16(a, w)
    assert_ulp(got, lin, 1, f"grouped gemm {M}")
    assert_ulp(_lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r), bf(lin.float() + r.float()), 2, f"grouped resid {M}", mag=lin)
    assert torch.equal(got, _lib.gemm_bf16(a, w)), "repeatable"


def test_gemm_strided_views():
    """Row-strided A (lda > K) and a row window of W - the restricted LM head uses both."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(0)
    abig = bf(torch.randn(300, 512, device="cuda"))
    wbig = bf(torch.randn(2048, 256, device="cuda") * 0.05)
    a = abig[:, 128:384]
    w = wbig[520:520 + 264]
    assert_ulp(_lib.gemm_bf16(a, w), ref_linear(a, w), 1, "strided gemm")


def test_gemm_residual_and_inplace():
    from mmada_parallel_b200 import _lib
    torch.manual_seed(1)
    a = bf(torch.randn(300, 768, device="cuda") * 0.5)
    w = bf(torch.randn(512, 768, device="cuda") * 0.05)
    r = bf(torch.randn(300, 512, device="cuda"))
    lin = ref_linear(a, w)
    want = bf(lin.float() + r.float())
    assert_ulp(_lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r), want, 2, "resid", mag=lin)
    r2 = r.clone()
    _lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r2, out=r2)
    assert_ulp(r2, want, 2, "resid in place", mag=lin)


def test_gemm_swiglu():
    from mmada_parallel_b200 import _lib
    torch.manual_seed(2)
    M, K, ff = 300, 512, 512
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w1 = bf(torch.randn(ff, K, device="cuda") * 0.08)
    w3 = bf(torch.randn(ff, K, device="cuda") * 0.08)
    wp = torch.empty(2 * ff, K, dtype=torch.bfloat16, device="cuda")
    wp.view(ff // 128, 2, 128, K)[:, 0] = w1.view(ff // 128, 128, K)
    wp.view(ff // 128, 2, 128, K)[:, 1] = w3.view(ff // 128, 128, K)
    got = _lib.gemm_bf16(a, wp, _lib.EPI_SWIGLU)
    want = bf(bf(torch.nn.functional.silu(ref_linear(a, w1).float())).float() * ref_linear(a, w3).float())
    assert got.shape == (M, ff)
    assert_ulp(got, want, 3, "swiglu")


def test_gemm_rejects_bad_arguments():
    from mmada_parallel_b200 import _lib
    a = bf(torch.randn(16, 60, device="cuda"))  # K not a multiple of 8
    w = bf(torch.randn(16, 60, device="cuda"))
    with pytest.raises(_lib.MmdpError):
        _lib.gemm_bf16(a, w)
    with pytest.raises(_lib.MmdpError):
        _lib.gemm_bf16(a.cpu(), w.cpu())  # no CPU fallback


@pytest.fixture(params=[6, 7])
def attn_version(request):
    """Both attention kernel generations of csrc/attention.cu (6: 128-key blocks, the default; 7: 64-key blocks, opt-in through
    MMDP_ATTN_VERSION / mmdp_set_option) run the same tests."""
    from mmada_parallel_b200 import _lib
    _lib.check(_lib.lib.mmdp_set_option(b"attn_version", request.param))
    yield request.param
    _lib.check(_lib.lib.mmdp_set_option(b"attn_version", 6))


def assert_attention_close(o, o_ref, what, ulps=4.0):
    """RELATIVE bound on the attention output against the fp32 softmax(QK^T)V reference. The kernel rounds P to bf16 before
    the PV product (relative 2^-9 per probability, averaging out over the row) and the output to bf16 (2^-9): the error of
    an element is bounded in bf16 ulps of max(|o|, rms(o) of its row) - elements that cancel to ~0 are measured against the
    row's typical magnitude. At L=2414 with random scores |o| ~ 0.03, so a kernel that is 10 % off fails by an order of
    magnitude (the round-1 bound, 2e-2 absolute, would have passed a 50 % error there)."""
    g, w = o.float(), o_ref.float()
    assert not torch.isnan(g).any(), what
    rms = w.pow(2).mean(-1, keepdim=True).sqrt()
    tol = ulps * torch.maximum(w.abs(), rms) * 2.0 ** -8
    bad = (g - w).abs() > tol
    rel = ((g - w).abs() / torch.maximum(w.abs(), rms)).max().item()
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} elements outside {ulps} bf16 ulp (max rel err {rel:.3e})"
    # and on average far inside it: mean error below half an ulp of the row magnitude
    assert ((g - w).abs() / rms).mean().item() < 0.5 * 2.0 ** -8, what


def ref_rope(t, cos, sin):
    tf = t.float()
    x1, x2 = tf[..., :64], tf[..., 64:]
    c, s = cos[:, None, :], sin[:, None, :]
    return bf(torch.cat([x1 * c + (-x2) * s, x2 * c + x1 * s], dim=-1))


@pytest.mark.parametrize("B,L,H", [(1, 128, 2), (2, 200, 2), (1, 640, 4), (3, 77, 2), (1, 2414, 4)])
def test_qkv_rope_and_attention(B, L, H, attn_version):
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import rope_tables
    torch.manual_seed(B * 1000 + L + H)
    d, M = H * 128, B * L
    a = bf(torch.randn(M, d, device="cuda"))
    wqkv = bf(torch.randn(3 * d, d, device="cuda") / math.sqrt(d))
    cos, sin = (t.cuda() for t in rope_tables(128, 500000.0, L))
    q, k, vt = _lib.qkv_rope(a, wqkv, H, L, cos, sin)
    qkv = ref_linear(a, wqkv)
    pos = torch.arange(M, device="cuda") % L
    q_ref = ref_rope(qkv[:, :d].view(M, H, 128), cos[pos], sin[pos]).view(M, d)
    k_ref = ref_rope(qkv[:, d:2 * d].view(M, H, 128), cos[pos], sin[pos]).view(M, d)
    def pair_mag(x):  # rotary mixes element i with i +- 64 of the same head: both magnitudes bound the rounding error
        xh = x.view(M, H, 2, 64).float().abs()
        return torch.maximum(xh[:, :, 0], xh[:, :, 1]).repeat(1, 1, 2).view(M, d)
    assert_ulp(q, q_ref, 2, "q rope", mag=pair_mag(qkv[:, :d]))
    assert_ulp(k, k_ref, 2, "k rope", mag=pair_mag(qkv[:, d:2 * d]))
    v_got = vt[..., :L].permute(0, 3, 1, 2).reshape(M, d)
    assert_ulp(v_got, qkv[:, 2 * d:], 1, "v^T")
    assert bool((vt[..., L:] == 0).all()), "pad columns of V^T must stay zero"
    scale = 1.0 / math.sqrt(128.0)
    o = _lib.attention(q, k, vt, B, H, L, scale)
    qh = q.view(B, L, H, 128).transpose(1, 2).float()
    kh = k.view(B, L, H, 128).transpose(1, 2).float()
    vh = v_got.reshape(B, L, H, 128).transpose(1, 2).float()
    o_ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(M, d)
    assert_attention_close(o, o_ref, f"attention B{B} L{L} H{H}")


def test_attention_lazy_rescale(attn_version):
    """The attention kernel against the fp32 reference, on random scores and on
    scores whose magnitude grows along the KV axis, so that the running row max jumps by far more than 2^8 in many KV
    blocks - the path that rescales the register-resident O accumulator."""
    from mmada_parallel_b200 import _lib
    scale = 1.0 / math.sqrt(128.0)
    version = attn_version
    try:
        for B, L, H, grow in [(2, 333, 2, 0.0), (1, 1000, 2, 60.0), (1, 129, 1, 200.0)]:
            torch.manual_seed(version * 100 + L)
            d, M = H * 128, B * L
            Lpad = (L + 7) // 8 * 8
            q = bf(torch.randn(M, d, device="cuda"))
            ramp = 1.0 + grow * (torch.arange(M, device="cuda") % L).float()[:, None] / L
            k = bf(torch.randn(M, d, device="cuda") * ramp)
            v = bf(torch.randn(M, d, device="cuda"))
            vt = torch.zeros(B, H, 128, Lpad, dtype=torch.bfloat16, device="cuda")
            vt[..., :L] = v.view(B, L, H, 128).permute(0, 2, 3, 1)
            o = _lib.attention(q, k, vt, B, H, L, scale)
            qh = q.view(B, L, H, 128).transpose(1, 2).float()
            kh = k.view(B, L, H, 128).transpose(1, 2).float()
            vh = v.view(B, L, H, 128).transpose(1, 2).float()
            o_ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(M, d)
            assert_attention_close(o, o_ref, f"attention v{version} L{L} grow{grow}")
    finally:
        pass


def test_attention_bitwise_repeatable(attn_version):
    """The same attention launch repeated many times at the full sequence length must be bitwise identical. (A parity wait
    that returns an mbarrier phase early lets a warpgroup read a K / V^T stage before its TMA load landed, or the producer
    overwrite one still in use - rare, timing dependent; this is the stress that exposes such races.) B=2."""
    from mmada_parallel_b200 import _lib
    B, L, H = 2, 2414, 16
    d, M, Lpad = H * 128, 2 * 2414, 2416
    torch.manual_seed(17)
    q = bf(torch.randn(M, d, device="cuda"))
    k = bf(torch.randn(M, d, device="cuda"))
    vt = torch.zeros(B, H, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    vt[..., :L] = bf(torch.randn(B, H, 128, L, device="cuda"))
    try:
        ref = _lib.attention(q, k, vt, B, H, L, 1.0 / math.sqrt(128.0)).clone()
        bad = 0
        for _ in range(150):
            bad += int(not torch.equal(_lib.attention(q, k, vt, B, H, L, 1.0 / math.sqrt(128.0)), ref))
        assert bad == 0, f"{bad} of 150 launches differ"
    finally:
        pass


def test_rmsnorm_embed_lfq():
    from mmada_parallel_b200 import _lib
    torch.manual_seed(3)
    for M, d in [(300, 4096), (17, 256)]:
        x = bf(torch.randn(M, d, device="cuda") * 3)
        w = bf(1 + 0.1 * torch.randn(d, device="cuda"))
        xf = x.float()
        want = w * bf(xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))
        assert_ulp(_lib.rmsnorm(x, w, 1e-5), want, 1, "rmsnorm")
        rows = torch.tensor([3, 1, M - 1, 0], dtype=torch.int32, device="cuda")
        assert_ulp(_lib.rmsnorm(x, w, 1e-5, rows=rows), want[rows.long()], 1, "rmsnorm rows")
    wte = bf(torch.randn(1000, 256, device="cuda"))
    ids = torch.randint(0, 1000, (77,), device="cuda")
    assert torch.equal(_lib.embed(ids, wte), wte[ids])
    vq = torch.randint(0, 8192, (2, 1024), device="cuda")
    from oracle.sampling import lfq_codebook_entry
    assert torch.equal(_lib.lfq_decode(vq, 13).cpu(), lfq_codebook_entry(vq.cpu(), 13))


def test_attention_full_length_relative_error(attn_version):
    """BASELINE sequence length, 32 heads (608 query tiles: four full waves of 132 SMs + a partial one) against
    the fp32 reference with the relative bound of assert_attention_close; also checks the split and unsplit tails agree."""
    from mmada_parallel_b200 import _lib
    B, L, H = 1, 2414, 32
    d, M, Lpad = H * 128, B * L, 2416
    torch.manual_seed(99)
    q = bf(torch.randn(M, d, device="cuda"))
    k = bf(torch.randn(M, d, device="cuda"))
    v = bf(torch.randn(M, d, device="cuda"))
    vt = torch.zeros(B, H, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    vt[..., :L] = v.view(B, L, H, 128).permute(0, 2, 3, 1)
    scale = 1.0 / math.sqrt(128.0)
    qh = q.view(B, L, H, 128).transpose(1, 2).float()
    kh = k.view(B, L, H, 128).transpose(1, 2).float()
    vh = v.view(B, L, H, 128).transpose(1, 2).float()
    o_ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(M, d)
    outs = []
    try:
        for split in (1, 0):
            _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", split))
            o = _lib.attention(q, k, vt, B, H, L, scale)
            assert_attention_close(o, o_ref, f"attention full length, split_tail={split}")
            outs.append(o.float())
    finally:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))
    # the two paths round P per KV block identically; only the merge of the split tiles differs (fp32 combine)
    assert (outs[0] - outs[1]).abs().max().item() <= 2.0 ** -8 * o_ref.abs().max().item()


@pytest.mark.parametrize("epi", ["qkv", "swiglu", "resid"])
def test_gemm_splitk_tail_matches_unsplit(epi):
    """Split-K tail (cooperative launch, fp32 partials reduced in fixed split order) vs the same kernel without the split,
    on the bench shapes (M=2414: 24 / 48 / 8 tail tiles): equal up to isolated 1-ulp roundings, repeatable bit for bit."""
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import rope_tables
    torch.manual_seed(11)
    M, K = 2414, 4096
    a = bf(torch.randn(M, K, device="cuda") * 0.5)

    def run():
        if epi == "qkv":
            H = K // 128
            w = bf(torch.randn(3 * K, K, device="cuda") / math.sqrt(K))
            cos, sin = (t.cuda() for t in rope_tables(128, 500000.0, M))
            return lambda: torch.cat([t.reshape(-1).float() for t in _lib.qkv_rope(a, w, H, M, cos, sin)])
        if epi == "swiglu":
            w = bf(torch.randn(24576, K, device="cuda") * 0.05)
            return lambda: _lib.gemm_bf16(a, w, _lib.EPI_SWIGLU).float()
        w = bf(torch.randn(4096, K, device="cuda") * 0.05)
        r = bf(torch.randn(M, 4096, device="cuda"))
        return lambda: _lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r).float()

    torch.manual_seed(12)
    fn = run()
    try:
        _lib.lib.mmdp_set_gemm_splitk(0)  # (the default 1-CTA kernel; the pair kernel has no split-K tail)
        ref = fn()
        _lib.lib.mmdp_set_gemm_splitk(3)  # split whenever a partial last wave exists
        got = fn()
        again = fn()
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
    assert torch.equal(got, again), "split-K tail must be deterministic"
    diff = (got - ref).abs()
    scale = ref.abs().max().item()
    assert diff.max().item() <= 2 * scale * 2.0 ** -8, (epi, diff.max().item())
    assert (got != ref).float().mean().item() < 0.02, (epi, (got != ref).float().mean().item())


@pytest.mark.parametrize("M,N,K", [(777, 1000, 520), (2414, 4096, 1024), (300, 512, 768)])
def test_gemm_pair_kernel_bit_identical_to_single(M, N, K):
    """The CTA-pair kernel (a 2-CTA cluster sharing the W tile by TMA multicast, opt-in through MMDP_GEMM_PAIR) accumulates K
    in the same order as the 1-CTA kernel without its split-K tail: plain, residual and SwiGLU epilogues must agree bit for bit."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M + K)
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    r = bf(torch.randn(M, N, device="cuda"))
    cases = [(_lib.EPI_PLAIN, {}), (_lib.EPI_RESID, dict(resid=r))]
    if N % 256 == 0:
        cases.append((_lib.EPI_SWIGLU, {}))
    try:
        _lib.lib.mmdp_set_gemm_splitk(0)
        for epi, kw in cases:
            _lib.lib.mmdp_set_gemm_pair(0)
            ref = _lib.gemm_bf16(a, w, epi, **kw)
            _lib.lib.mmdp_set_gemm_pair(1)
            got = _lib.gemm_bf16(a, w, epi, **kw)
            assert torch.equal(got, ref), epi
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.lib.mmdp_set_gemm_pair(0)
