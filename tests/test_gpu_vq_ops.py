"""Op-level tests of the VQ tokenizers' kernels (csrc/conv_tf32.cu, csrc/vq_codebook.cu) against torch fp64 restatements of
the same operations. The network-level tests (test_gpu_magvit.py, test_gpu_vqmodel.py) bound a whole decode at 0.02
absolute, loose enough to hide one piece being subtly wrong; here every kernel is checked alone, at the MagViT / aMUSEd
production shapes and at edge shapes, through the test hooks of include/mmdp_testing.h.

Stated tolerances (u = 2^-24, the fp32 unit roundoff):
  - TF32 convolution, against the fp64 conv of the fp32 operands. tf32 wgmma keeps 10 explicit mantissa bits of each
    operand, a relative error below 2^-10 per operand and 2^-9 per product; the products are accumulated in fp32. Two checks:
      per element   |got - ref| <= 2^-8 * sum_k |a_k w_k|  (+ 4u of the epilogue's |ref| + |bias| + |R|)
                    2^-9 for the operands, the other 2^-9 covers the fp32 accumulation (|err| <= n u sum|.| with n <= 6912);
      statistical   rms(got - ref) <= 2 * 2^-10 * rms(sqrt(sum_k (a_k w_k)^2))
                    the per-product error is a_k w_k e_k with e_k in [0, 2^-9): its mean (<= 2^-10 if truncated, 0 if rounded)
                    scales sum a_k w_k, whose rms equals rms(sqrt(sum (a w)^2)) for the zero-mean test data, and its spread
                    adds sqrt(E[(e - Ee)^2]) <= 2^-10 / sqrt(3) of the same; c = 2 leaves ~1.6x over 1.15 * 2^-10.
    A 32-channel k-block dropped from 6912 terms moves a value by ~sqrt(32 / 6912) = 2^-3.9 of that rms: far inside the
    per-element bound, 20x outside the statistical one.
  - The same against an fp64 reference whose operands were truncated to TF32 (what the hardware reads, see pack_conv_kernel):
    only accumulation error remains, per element <= (n_k / 8 + 8) 2^-20 sum|a w| (n_k / 8 wgmma steps, each rounding the fp32
    accumulator and adding 8 products) and rms <= 2^-13 rms(sqrt(sum (a w)^2)). Operands rounded to nearest instead of
    truncated would differ from this reference by ~2^-11.5 of that rms and fail; the test prints the error against both
    models.
  - GroupNorm: fp32 evaluation of (x - mean) rstd gamma + beta from statistics exact to 2^-16 (the mean to 2^-16 of the
    group's deviation, rstd to 2^-16 relative; the fp32 per-thread sums of ~130 terms of x - pivot, each a few deviations
    large, carry ~sqrt(130) u of a few deviations = 2^-18):
        |got - ref| <= |gamma| 2^-16 (1 + |n|) + |gamma| rstd 4u (|mean| + |x - mean|) + 4u (|gamma n| + |beta|)   (n = normalised x)
    (SiLU: x 1.1, its slope bound, plus 8u |ref|). The only offset-dependent term is the fp32 rounding of the mean itself,
    4u |mean| rstd, which torch's fp32 GroupNorm carries as well; nothing grows with (mean / std)^2, which is what a variance
    taken as E[x^2] - mean^2 in fp32 does.
  - softmax: exp(s - max) with s - max rounded (u |s - max| relative), the fp32 sum of n / 256 + 8 terms and the division:
        |got - ref| <= ref u (|s - max| + n / 256 + 16) + 2^-126.
  - layout kernels, LFQ, codebook gather, nearest-code ids and z_q: bit-exact (they move or compare values, no arithmetic).
"""
import ctypes as C
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from helpers import ROOT

gpu = pytest.mark.gpu
SENT = -7777.0  # sentinel of memory a kernel must not write

_vp, _i, _i64, _f, _ll = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_longlong
# name -> argtypes (every hook returns int); must list every symbol declared in include/mmdp_testing.h
HOOKS = {
    "mmdp_testing_conv_tf32": [_vp, _i, _ll, _vp, _i, _i, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _i, _f, _i, _i, _i, _i, _vp],
    "mmdp_testing_gn_swish": [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _f, _i, _i, _vp],
    "mmdp_testing_upsample2x": [_vp, _vp, _i, _i, _i, _i, _vp],
    "mmdp_testing_downsample_pick": [_vp, _vp, _i, _i, _i, _i, _vp],
    "mmdp_testing_softmax_rows_ld": [_vp, _i, _i, _i, _vp],
    "mmdp_testing_zero_border": [_vp, _i, _i, _i, _i, _vp],
    "mmdp_testing_nchw_to_padded": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "mmdp_testing_padded_to_nchw": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "mmdp_testing_lfq_to_padded": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "mmdp_testing_lfq_indices": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "mmdp_testing_codebook_to_padded": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i64, _vp, _vp],
}


def declared_testing_symbols():
    src = open(os.path.join(ROOT, "include", "mmdp_testing.h")).read()
    return sorted(set(re.findall(r"MMDP_API[^;(]*?\b(mmdp_[a-z0-9_]+)\s*\(", src)))


def hooks():
    """libmmdp.so with the argument types of the test hooks set."""
    from mmada_parallel_b200 import _lib
    for name, args in HOOKS.items():
        fn = getattr(_lib.lib, name)
        fn.restype, fn.argtypes = _i, args
    return _lib.lib


def call(name, *args):
    from mmada_parallel_b200 import _lib
    rc = getattr(hooks(), name)(*args, _lib.stream_ptr())
    _lib.check(rc)


def p(t):
    return None if t is None else t.data_ptr()


def r32(c):
    return (c + 31) // 32 * 32


def padded(x, cpad, border=0.0):
    """NCHW [B, C, H, W] -> padded channels-last [B * (H+2) * (W+2), cpad]: zero channels >= C, border pixels = `border`."""
    B, Cc, H, W = x.shape
    y = F.pad(x.permute(0, 2, 3, 1), (0, cpad - Cc, 1, 1, 1, 1))
    if border != 0.0:
        y[:, 0], y[:, -1], y[:, :, 0], y[:, :, -1] = border, border, border, border
    return y.reshape(B * (H + 2) * (W + 2), cpad).contiguous()


def interior(y, B, H, W, c=None):
    """padded rows [B * (H+2) * (W+2), ld] -> [B, H, W, c]"""
    v = y.view(B, H + 2, W + 2, -1)[:, 1:H + 1, 1:W + 1]
    return v if c is None else v[..., :c]


def border_mask(B, H, W, device):
    m = torch.ones(B, H + 2, W + 2, dtype=torch.bool, device=device)
    m[:, 1:H + 1, 1:W + 1] = False
    return m.reshape(-1)


def tf32_trunc(x):
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_rna(x):
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def rms(t):
    return float(t.double().pow(2).mean().sqrt())


# ------------------------------------------------------------------------------------------------------------------
# convolution bounds
# ------------------------------------------------------------------------------------------------------------------
def conv_check(got, ref, absb, sq, epi, k_total, ref_t=None):
    """(ok, report) for a TF32 conv output against its fp64 reference (module docstring). absb = alpha * sum|a w|,
    sq = alpha^2 sum (a w)^2, epi = |bias| + |R| of the epilogue, ref_t = fp64 reference of the TF32-truncated operands."""
    got, ref = got.double(), ref.double()
    if not torch.isfinite(got).all():
        return False, "non-finite output"
    err = (got - ref).abs()
    tol = 2.0 ** -8 * absb + 4 * 2.0 ** -24 * (ref.abs() + epi)
    spread = rms(sq.sqrt())
    e_rms, b_rms = rms(got - ref), 2 * 2.0 ** -10 * spread
    rep = {"max_err/bound": float((err / tol).max()), "rms_err": e_rms, "rms_bound": b_rms}
    ok = bool((err <= tol).all()) and e_rms <= b_rms
    if ref_t is not None:
        et = (got - ref_t.double()).abs()
        tol_t = (k_total / 8 + 8) * 2.0 ** -20 * absb + 4 * 2.0 ** -24 * (ref.abs() + epi)
        bt = 2.0 ** -13 * spread + 4 * 2.0 ** -24 * rms(ref.abs() + epi)
        rep.update({"tf32_max_err/bound": float((et / tol_t).max()), "tf32_rms_err": rms(got - ref_t.double()), "tf32_rms_bound": bt})
        ok = ok and bool((et <= tol_t).all()) and rep["tf32_rms_err"] <= bt
    return ok, rep


def assert_conv(got, ref, absb, sq, epi, k_total, what, ref_t=None, ref_rn=None):
    ok, rep = conv_check(got, ref, absb, sq, epi, k_total, ref_t)
    if ref_rn is not None:
        rep["rms_err_vs_round_to_nearest_model"] = rms(got.double() - ref_rn.double())
    print(f"[{what}] " + (", ".join(f"{k} {v:.3e}" for k, v in rep.items()) if isinstance(rep, dict) else rep))
    assert ok, (what, rep)


def conv_ref(x, w, bias, alpha, pad):
    """fp64 alpha * conv(x, w) + bias, |.|-sum and square-sum of the products (NCHW in, NHWC out)"""
    xd, wd = x.double(), w.double()
    out = alpha * F.conv2d(xd, wd, padding=pad)
    absb = abs(alpha) * F.conv2d(xd.abs(), wd.abs(), padding=pad)
    sq = alpha * alpha * F.conv2d(xd * xd, wd * wd, padding=pad)
    if bias is not None:
        out = out + bias.double()[None, :, None, None]
    return out.permute(0, 2, 3, 1), absb.permute(0, 2, 3, 1), sq.permute(0, 2, 3, 1)


def pack_w(w, kpad):
    """OIHW -> [tap][cout][kpad] (pack_conv_kernel's layout)"""
    co, ci, k, _ = w.shape
    return F.pad(w.permute(2, 3, 0, 1).reshape(k * k, co, ci), (0, kpad - ci)).contiguous()


def run_conv_padded(x, w, bias=None, R=None, alpha=1.0, ldc=None, wpack=None):
    """conv_tf32 over padded NHWC images the way Fwd::conv launches it; returns the full output buffer [M, ldc]."""
    B, cin, H, W = x.shape
    cout, k = w.shape[0], w.shape[2]
    kpad, Hp, Wp = r32(cin), H + 2, W + 2
    M = B * Hp * Wp
    A = padded(x, kpad)
    wp = pack_w(w, kpad) if wpack is None else wpack
    T = k * k
    sh = [(ky - 1) * Wp + (kx - 1) for ky in range(3) for kx in range(3)] if k == 3 else [0]
    shifts = (C.c_int * T)(*sh)
    ldc = ldc or r32(cout)
    out = torch.full((M, ldc), SENT, device=x.device)
    call("mmdp_testing_conv_tf32", p(A), kpad, M, p(wp), M, cout, kpad, T, shifts, p(out), ldc, p(R), ldc if R is not None else 0,
         p(bias), 0, alpha, Wp, Hp, 0, 0)
    return out


def conv_case(cin, cout, H, W, B, k, bias=True, resid=False, alpha=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, cin, H, W, device="cuda", generator=g)
    w = torch.randn(cout, cin, k, k, device="cuda", generator=g) / math.sqrt(cin * k * k)
    b = torch.randn(cout, device="cuda", generator=g) if bias else None
    ldc = r32(cout)
    R = None
    if resid:
        R = torch.randn(B * (H + 2) * (W + 2), ldc, device="cuda", generator=g)
    out = run_conv_padded(x, w, b, R, alpha)
    return x, w, b, R, out


CONV_CASES = [  # cin, cout, H, W, B, k, bias, resid, alpha
    (3, 128, 32, 32, 1, 3, True, False, 1.0),     # encoder conv_in: cin padded to 32
    (13, 512, 1, 1, 1, 3, True, False, 1.0),      # 1x1 grid: every tap but the centre reads the border
    (64, 3, 1, 37, 3, 3, True, False, 1.0),       # conv_out-like cout 3, B = 3 (taps cross into neighbour images)
    (128, 13, 37, 1, 3, 3, True, True, 1.0),
    (256, 200, 5, 7, 3, 3, True, True, 0.37),     # partial n-tile, residual, alpha
    (512, 512, 32, 32, 1, 3, True, True, 1.0),    # MagViT mid / aMUSEd production
    (768, 768, 64, 16, 1, 3, True, False, 1.0),   # aMUSEd deepest level (K = 6912)
    (768, 64, 5, 7, 3, 3, False, False, 1.0),
    (13, 13, 32, 32, 1, 1, True, False, 1.0),     # post_quant_conv
    (512, 768, 37, 1, 3, 1, True, True, 1.0),     # 1x1 shortcut
    (128, 256, 64, 16, 1, 1, True, False, 2.0),
    (64, 200, 1, 1, 3, 1, False, True, 1.0),
]


@gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "x".join(map(str, c[:6])) + ("b" if c[6] else "") + ("r" if c[7] else "")
                         + ("a" if c[8] != 1.0 else ""))
def test_conv_tf32_vs_fp64(case):
    cin, cout, H, W, B, k, bias, resid, alpha = case
    x, w, b, R, out = conv_case(cin, cout, H, W, B, k, bias, resid, alpha, seed=cin * 7 + cout)
    ref, absb, sq = conv_ref(x, w, b, alpha, k // 2)
    ref_t, _, _ = conv_ref(tf32_trunc(x), tf32_trunc(w), b, alpha, k // 2)
    ref_rn, _, _ = conv_ref(tf32_rna(x), tf32_rna(w), b, alpha, k // 2)
    epi = torch.zeros_like(ref)
    if b is not None:
        epi = epi + b.double().abs()
    if R is not None:
        Ri = interior(R, B, H, W, cout).double()
        ref, ref_t, ref_rn, epi = ref + Ri, ref_t + Ri, ref_rn + Ri, epi + Ri.abs()
    got = interior(out, B, H, W, cout)
    assert_conv(got, ref, absb, sq, epi, k * k * r32(cin), f"conv {case}", ref_t=ref_t, ref_rn=ref_rn)
    bm = border_mask(B, H, W, out.device)
    assert (out[bm, :cout] == 0).all(), "border rows must be written as zero"
    assert (out[:, cout:] == SENT).all(), "columns [N, ldc) must not be written"


@gpu
def test_conv_bounds_reject_plausible_bugs():
    """Negative controls: the kernel's output with the effect of one plausible bug added (computed in fp64 from the
    reference) must fail conv_check, while the output itself passes."""
    cin, cout, H, W, B = 512, 200, 16, 12, 2
    x, w, b, R, out = conv_case(cin, cout, H, W, B, 3, True, True, 1.0, seed=5)
    ref, absb, sq = conv_ref(x, w, b, 1.0, 1)
    Ri = interior(R, B, H, W, cout).double()
    ref = ref + Ri
    epi = b.double().abs() + Ri.abs()
    got = interior(out, B, H, W, cout).double()
    kt = 9 * cin
    assert conv_check(got, ref, absb, sq, epi, kt)[0]

    w_tap = w.clone()
    w_tap[:, :, 0, 2] = 0  # one tap zeroed
    w_blk = w.clone()
    w_blk[:, 64:96, 1, 1] = 0  # one 32-channel k-block of the centre tap zeroed
    R_sh = torch.roll(R, 1, dims=0)  # residual read one row off
    bugs = {
        "tap zeroed": conv_ref(x, w_tap, b, 1.0, 1)[0] + Ri,
        "k-block zeroed": conv_ref(x, w_blk, b, 1.0, 1)[0] + Ri,
        "bias dropped": conv_ref(x, w, None, 1.0, 1)[0] + Ri,
        "residual shifted one row": conv_ref(x, w, b, 1.0, 1)[0] + interior(R_sh, B, H, W, cout).double(),
    }
    for name, ref_bug in bugs.items():
        ok, rep = conv_check(got + (ref_bug - ref), ref, absb, sq, epi, kt)
        print(f"[negative control: {name}] rejected={not ok} {rep}")
        assert not ok, f"the bounds accept a kernel with '{name}'"


@gpu
def test_conv_tf32_compact_and_scatter_modes():
    """T = 1 compact products of the mid-block attention: V^T = Wv . h^T with the bias along m (ldc = round32(hw) > N),
    and proj_out scattered into the padded layout with a padded residual (border rows untouched)."""
    g = torch.Generator(device="cuda").manual_seed(11)
    for Cc, H, W in ((512, 20, 20), (768, 24, 24), (64, 1, 37)):
        hw, hwp = H * W, r32(H * W)
        hn = torch.randn(hw, Cc, device="cuda", generator=g)
        wv = torch.randn(Cc, Cc, device="cuda", generator=g) / math.sqrt(Cc)
        bv = torch.randn(Cc, device="cuda", generator=g)
        vt = torch.full((Cc, hwp), SENT, device="cuda")
        call("mmdp_testing_conv_tf32", p(wv), Cc, Cc, p(hn), Cc, hw, Cc, 1, None, p(vt), hwp, None, 0, p(bv), 1, 1.0, 0, 0, 0, 0)
        wd, hd = wv.double(), hn.double()
        ref = wd @ hd.t() + bv.double()[:, None]
        ref_t = tf32_trunc(wv).double() @ tf32_trunc(hn).double().t() + bv.double()[:, None]
        assert_conv(vt[:, :hw], ref, wd.abs() @ hd.abs().t(), (wd * wd) @ (hd * hd).t(), bv.double().abs()[:, None].expand_as(ref),
                    r32(Cc), f"V^T C={Cc} hw={hw}", ref_t=ref_t)
        assert (vt[:, hw:] == SENT).all()

        B = 2
        o = torch.randn(B * hw, Cc, device="cuda", generator=g)
        wp = torch.randn(Cc, Cc, device="cuda", generator=g) / math.sqrt(Cc)
        bp = torch.randn(Cc, device="cuda", generator=g)
        X = torch.randn(B * (H + 2) * (W + 2), Cc, device="cuda", generator=g)
        Y = torch.full_like(X, SENT)
        call("mmdp_testing_conv_tf32", p(o), Cc, B * hw, p(wp), B * hw, Cc, Cc, 1, None, p(Y), Cc, p(X), Cc, p(bp), 0, 1.0, 0, 0, W, H)
        od, wpd = o.double(), wp.double()
        Xi = interior(X, B, H, W).reshape(B * hw, Cc).double()
        ref = od @ wpd.t() + bp.double() + Xi
        ref_t = tf32_trunc(o).double() @ tf32_trunc(wp).double().t() + bp.double() + Xi
        assert_conv(interior(Y, B, H, W).reshape(B * hw, Cc), ref, od.abs() @ wpd.abs().t(), (od * od) @ (wpd * wpd).t(),
                    bp.double().abs() + Xi.abs(), r32(Cc), f"proj_out scatter C={Cc} {H}x{W}", ref_t=ref_t)
        assert (Y[border_mask(B, H, W, Y.device)] == SENT).all(), "the scatter writes interior rows only"


# ------------------------------------------------------------------------------------------------------------------
# mid-block attention composite
# ------------------------------------------------------------------------------------------------------------------
class AttnBuffers:
    def __init__(self, B, C, max_hw, max_H, max_W):
        f = lambda *s: torch.full(s, float("nan"), device="cuda")  # noqa: E731  stale garbage until written
        self.T = f(B * max_hw * C)
        self.q, self.k, self.o = f(B * max_hw, C), f(B * max_hw, C), f(B * max_hw, C)
        self.vt = f(C * r32(max_hw))
        self.s = f(max_hw * r32(max_hw))
        self.Y = f(B * (max_H + 2) * (max_W + 2) * C)
        self.stats = torch.zeros(B * 64, dtype=torch.float64, device="cuda")


def attn_native(bf, X, wts, B, C, H, W):
    """Fwd::attn (vq_decoder.cu) restated over the hooks"""
    gn_g, gn_b, wq, bq, wk, bk, wv, bv, wp, bp = wts
    hw, hwp = H * W, r32(H * W)
    call("mmdp_testing_gn_swish", p(X), p(bf.T), B, C, H, W, p(bf.stats), p(gn_g), p(gn_b), 1e-6, 0, 1)
    call("mmdp_testing_conv_tf32", p(bf.T), C, B * hw, p(wq), B * hw, C, C, 1, None, p(bf.q), C, None, 0, p(bq), 0, 1.0, 0, 0, 0, 0)
    call("mmdp_testing_conv_tf32", p(bf.T), C, B * hw, p(wk), B * hw, C, C, 1, None, p(bf.k), C, None, 0, p(bk), 0, 1.0, 0, 0, 0, 0)
    scale = 1.0 / math.sqrt(C)
    if hwp != hw:
        bf.s[:hw * hwp].zero_()
        bf.vt[:C * hwp].zero_()
    for b in range(B):
        hn = bf.T[b * hw * C:]
        call("mmdp_testing_conv_tf32", p(wv), C, C, p(hn), C, hw, C, 1, None, p(bf.vt), hwp, None, 0, p(bv), 1, 1.0, 0, 0, 0, 0)
        call("mmdp_testing_conv_tf32", p(bf.q[b * hw:]), C, hw, p(bf.k[b * hw:]), hw, hw, C, 1, None, p(bf.s), hwp, None, 0, None, 0,
             scale, 0, 0, 0, 0)
        call("mmdp_testing_softmax_rows_ld", p(bf.s), hw, hw, hwp)
        call("mmdp_testing_conv_tf32", p(bf.s), hwp, hw, p(bf.vt), hw, C, hwp, 1, None, p(bf.o[b * hw:]), C, None, 0, None, 0, 1.0, 0,
             0, 0, 0)
    call("mmdp_testing_conv_tf32", p(bf.o), C, B * hw, p(wp), B * hw, C, C, 1, None, p(bf.Y), C, p(X), C, p(bp), 0, 1.0, 0, 0, W, H)
    call("mmdp_testing_zero_border", p(bf.Y), B, C, H, W)
    return bf.Y[:B * (H + 2) * (W + 2) * C].view(B * (H + 2) * (W + 2), C)


def attn_ref_and_bound(x, wts, B, C, H, W):
    """fp64 single-head attention block, a per-element worst-case bound and a per-element error spread, both propagated
    through the stages.
      worst case: every TF32 product costs 2^-8 sum|a b| (the conv bound), an error e_S of the scores moves a probability by
        at most P (exp(2 max_row e_S) - 1), and the input errors of each product are carried by |.| products;
      spread: every TF32 product adds 2 * 2^-10 sqrt(sum (a b)^2) (the conv statistical bound), input errors are independent
        and add in quadrature (sqrt(e_a^2 . b^2)), and dP = P (dS - E_P[dS]) gives e_P^2 = P^2 (e_S^2 + E_P[e_S^2]); the
        coherent part of the truncation (a shrink of the scores) passes the softmax with a sign and is added linearly."""
    gn_g, gn_b, wq, bq, wk, bk, wv, bv, wp, bp = [t.double() for t in wts]
    hw = H * W
    xd = x.double().permute(0, 2, 3, 1).reshape(B, hw, C)
    xg = xd.view(B, hw, 32, C // 32)
    mu = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
    h = ((xg - mu) / torch.sqrt(var + 1e-6)).view(B, hw, C) * gn_g + gn_b
    eh = 2.0 ** -16 * (h.abs() + gn_b.abs())
    u8, s9 = 2.0 ** -8, 2.0 ** -9
    T = lambda t: t.transpose(-1, -2)  # noqa: E731

    def lin(a, ea, sa, w, bias):
        """a @ w^T + bias with (worst-case, spread) errors from input errors (ea, sa)"""
        return (a @ T(w) + bias, u8 * a.abs() @ T(w.abs()) + ea @ T(w.abs()),
                torch.sqrt(s9 ** 2 * (a * a) @ T(w * w) + (sa * sa) @ T(w * w)))

    q, eq, sq = lin(h, eh, eh, wq, bq)
    k, ek, sk = lin(h, eh, eh, wk, bk)
    v, ev, sv = lin(h, eh, eh, wv, bv)
    sc = 1.0 / math.sqrt(C)
    S = sc * q @ T(k)
    eS = sc * (u8 * q.abs() @ T(k.abs()) + eq @ T(k.abs()) + q.abs() @ T(ek))
    sS = sc * torch.sqrt(s9 ** 2 * (q * q) @ T(k * k) + (sq * sq) @ T(k * k) + (q * q) @ T(sk * sk))
    P = torch.softmax(S, dim=-1)
    eP = P * torch.expm1(2 * eS.amax(-1, keepdim=True)) + 2.0 ** -20 * P
    sP = P * torch.sqrt(sS * sS + (P * sS * sS).sum(-1, keepdim=True)) + 2.0 ** -20 * P
    O = P @ v
    eO = u8 * P @ v.abs() + eP @ v.abs() + P @ ev
    # truncated operands shrink q, k and S coherently, each by a mean relative factor below 2^-9: S by up to 3 * 2^-9 S, which
    # moves O by 3 * 2^-9 Cov_P(S, v) in one direction (not independent across the keys: added linearly)
    coh = 3 * s9 * (P * (S - (P * S).sum(-1, keepdim=True))) @ v
    sO = torch.sqrt(s9 ** 2 * (P * P) @ (v * v) + (sP * sP) @ (v * v) + (P * P) @ (sv * sv)) + coh.abs()
    out, eout, sout = lin(O, eO, sO, wp, bp)
    out = out + xd
    eout = eout + 4 * 2.0 ** -24 * (out.abs() + xd.abs())
    return out, eout, sout


def attn_weights(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    s = 1 / math.sqrt(C)
    return [1 + 0.1 * r(C), 0.1 * r(C), r(C, C) * s, 0.1 * r(C), r(C, C) * s, 0.1 * r(C), r(C, C) * s, 0.1 * r(C), r(C, C) * s, 0.1 * r(C)]


@gpu
def test_mid_block_attention_composite():
    """compact GN -> q, k, V^T -> scaled S -> softmax_rows_ld -> P.V over round32(hw) keys -> scattered proj_out + residual ->
    zero_border, against fp64 attention. hw = 576 (no key padding) runs first on the same buffers, then hw = 400 (padded to
    416, the padding columns of S and V^T are read and hold the larger grid's values until re-zeroed)."""
    C, B = 512, 2
    wts = attn_weights(C, 3)
    bf = AttnBuffers(B, C, 576, 24, 24)
    g = torch.Generator(device="cuda").manual_seed(4)
    for H, W in ((24, 24), (20, 20)):
        x = torch.randn(B, C, H, W, device="cuda", generator=g) * 1.5 + 0.3
        X = padded(x, C)
        Y = attn_native(bf, X, wts, B, C, H, W)
        ref, eb, spread = attn_ref_and_bound(x, wts, B, C, H, W)
        got = interior(Y, B, H, W).reshape(B, H * W, C).double()
        err = (got - ref).abs()
        branch = ref - x.double().permute(0, 2, 3, 1).reshape(B, H * W, C)
        print(f"[attention {H}x{W} C={C}] max err {float(err.max()):.3e}, max err/bound {float((err / eb).max()):.3e}, "
              f"rms err {rms(got - ref):.3e}, rms bound {rms(spread):.3e} (rms of the attention branch {rms(branch):.3e})")
        assert torch.isfinite(Y).all()
        assert (Y[border_mask(B, H, W, Y.device)] == 0).all()
        assert (err <= eb).all()
        assert rms(got - ref) <= rms(spread)


# ------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ------------------------------------------------------------------------------------------------------------------
def gn_ref(x, gamma, beta, eps, swish):
    """fp64 GroupNorm(32) (+ SiLU) of NCHW x; returns (y, bound) in NHWC."""
    B, Cc, H, W = x.shape
    xd = x.double().view(B, 32, -1)
    mu = xd.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    n = ((xd - mu) * rstd).view(B, Cc, H, W)
    gd, bd = gamma.double()[None, :, None, None], beta.double()[None, :, None, None]
    t = n * gd + bd
    u = 2.0 ** -24
    mu4, rs4 = mu.view(B, 32, 1, 1, 1).expand(B, 32, Cc // 32, H, W).reshape(B, Cc, H, W), \
        rstd.view(B, 32, 1, 1, 1).expand(B, 32, Cc // 32, H, W).reshape(B, Cc, H, W)
    bound = (gd.abs() * 2.0 ** -16 * (1 + n.abs()) + gd.abs() * rs4 * 4 * u * (mu4.abs() + (x.double() - mu4).abs())
             + 4 * u * ((gd * n).abs() + bd.abs()))
    if swish:
        t = t * torch.sigmoid(t)
        bound = 1.1 * bound + 8 * u * t.abs()
    return t.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)


def run_gn(x, gamma, beta, swish, compact):
    B, Cc, H, W = x.shape
    X = padded(x, Cc, border=float("nan"))  # the border is never read
    rows = B * H * W if compact else B * (H + 2) * (W + 2)
    Y = torch.full((rows, Cc), float("nan"), device="cuda")
    stats = torch.full((B * 64,), float("nan"), dtype=torch.float64, device="cuda")
    call("mmdp_testing_gn_swish", p(X), p(Y), B, Cc, H, W, p(stats), p(gamma), p(beta), 1e-6, int(swish), int(compact))
    return Y


# C 32: one channel per group; 384: TC = 96 (idle pixel lanes); 1024: C4 = 256; 2048: two c4 per thread; 128 at 512x512:
# the full-resolution aMUSEd level; 520x520: more than 16 chunks per SM, the chunk count is capped (uneven chunks)
GN_SHAPES = [(32, 1, 1), (128, 3, 5), (384, 32, 32), (768, 32, 32), (1024, 3, 5), (2048, 1, 1), (2048, 32, 32), (128, 512, 512),
             (64, 520, 520)]


@gpu
@pytest.mark.parametrize("C_,H,W", GN_SHAPES)
@pytest.mark.parametrize("offset", [0, 30, 1000])
def test_group_norm_vs_fp64(C_, H, W, offset):
    B = 3
    g = torch.Generator(device="cuda").manual_seed(C_ + H + offset)
    std = torch.tensor([0.5, 2.0, 7.0], device="cuda")[:, None, None, None]
    ch = 1 + 0.2 * torch.randn(1, C_, 1, 1, device="cuda", generator=g)  # channels differ inside a group
    x = (torch.randn(B, C_, H, W, device="cuda", generator=g) * ch + offset) * std
    x[1] += 0.5 * std[1]  # a different mean per image
    gamma = 1 + 0.5 * torch.randn(C_, device="cuda", generator=g)
    beta = 0.5 * torch.randn(C_, device="cuda", generator=g)
    for swish, compact in ((True, False), (False, True), (False, False)):
        if H * W > 4096 and (swish, compact) != (True, False):
            continue
        Y = run_gn(x, gamma, beta, swish, compact)
        ref, bound = gn_ref(x, gamma, beta, 1e-6, swish)
        got = Y.view(B, H, W, C_) if compact else interior(Y, B, H, W)
        err = (got.double() - ref).abs()
        print(f"[group norm C={C_} {H}x{W} mean/std={offset} swish={int(swish)} compact={int(compact)}] max err {float(err.max()):.3e} "
              f"max err/bound {float((err / bound).max()):.3e}")
        assert torch.isfinite(got).all()
        assert (err <= bound).all(), f"max err/bound {float((err / bound).max()):.3e}"
        if not compact:
            assert (Y[border_mask(B, H, W, Y.device)] == 0).all(), "the padded border must be written as zero"


# ------------------------------------------------------------------------------------------------------------------
# layout and small kernels (bit-exact)
# ------------------------------------------------------------------------------------------------------------------
@gpu
def test_upsample_and_zero_border():
    g = torch.Generator(device="cuda").manual_seed(1)
    for Cc, H, W, B in ((128, 5, 7, 3), (512, 32, 32, 1), (4, 1, 1, 2)):
        x = torch.randn(B, Cc, H, W, device="cuda", generator=g)
        X = padded(x, Cc, border=float("nan"))
        Y = torch.full((B * (2 * H + 2) * (2 * W + 2), Cc), float("nan"), device="cuda")
        call("mmdp_testing_upsample2x", p(X), p(Y), B, Cc, H, W)
        want = x.repeat_interleave(2, 2).repeat_interleave(2, 3).permute(0, 2, 3, 1)
        assert torch.equal(interior(Y, B, 2 * H, 2 * W), want)
        assert (Y[border_mask(B, 2 * H, 2 * W, Y.device)] == 0).all()

        Z = torch.randn(B * (H + 2) * (W + 2), Cc, device="cuda", generator=g)
        Z0 = Z.clone()
        call("mmdp_testing_zero_border", p(Z), B, Cc, H, W)
        bm = border_mask(B, H, W, Z.device)
        assert (Z[bm] == 0).all() and torch.equal(Z[~bm], Z0[~bm])


@gpu
def test_downsample_pick_and_stride2_conv():
    g = torch.Generator(device="cuda").manual_seed(2)
    for Cc, H, W, B in ((128, 8, 6, 3), (256, 64, 64, 1), (4, 2, 2, 1)):
        src = torch.randn(B * (H + 2) * (W + 2), Cc, device="cuda", generator=g)
        dst = torch.full((B * (H // 2 + 2) * (W // 2 + 2), Cc), float("nan"), device="cuda")
        call("mmdp_testing_downsample_pick", p(src), p(dst), B, Cc, H, W)
        assert torch.equal(interior(dst, B, H // 2, W // 2), interior(src, B, H, W)[:, 1::2, 1::2])
        assert (dst[border_mask(B, H // 2, W // 2, dst.device)] == 0).all()
    # Downsample: F.pad(x, (0, 1, 0, 1)) + 3x3 stride-2 conv == the stride-1 zero-border conv picked at odd pixels
    for cin, cout, H, W, B in ((128, 128, 16, 12, 2), (512, 512, 64, 64, 1)):
        x = torch.randn(B, cin, H, W, device="cuda", generator=g)
        w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g) / math.sqrt(9 * cin)
        b = torch.randn(cout, device="cuda", generator=g)
        full = run_conv_padded(x, w, b)
        dst = torch.full((B * (H // 2 + 2) * (W // 2 + 2), cout), float("nan"), device="cuda")
        call("mmdp_testing_downsample_pick", p(full), p(dst), B, cout, H, W)
        xp = F.pad(x.double(), (0, 1, 0, 1))
        ref = (F.conv2d(xp, w.double(), b.double(), stride=2)).permute(0, 2, 3, 1)
        absb = F.conv2d(xp.abs(), w.double().abs(), stride=2).permute(0, 2, 3, 1)
        sq = F.conv2d(xp * xp, w.double() ** 2, stride=2).permute(0, 2, 3, 1)
        assert_conv(interior(dst, B, H // 2, W // 2), ref, absb, sq, b.double().abs().expand_as(ref), 9 * cin,
                    f"downsample conv {cin}->{cout} {H}x{W}")


@gpu
def test_nchw_padded_round_trip():
    g = torch.Generator(device="cuda").manual_seed(3)
    for Cc, Cpad, H, W, B in ((3, 32, 17, 9, 3), (13, 32, 1, 1, 2), (64, 96, 8, 8, 1)):
        x = torch.randn(B, Cc, H, W, device="cuda", generator=g)
        Y = torch.full((B * (H + 2) * (W + 2), Cpad), float("nan"), device="cuda")
        call("mmdp_testing_nchw_to_padded", p(x), p(Y), B, Cc, Cpad, H, W)
        assert torch.equal(Y, padded(x, Cpad))
        back = torch.full_like(x, float("nan"))
        call("mmdp_testing_padded_to_nchw", p(Y), p(back), B, Cc, Cpad, H, W)
        assert torch.equal(back, x)


@gpu
def test_lfq_round_trip():
    from oracle.sampling import lfq_codebook_entry
    g = torch.Generator(device="cuda").manual_seed(4)
    bits, Cpad = 13, 32
    for B, H, W in ((2, 16, 16), (1, 1, 1), (3, 5, 37)):
        ids = torch.randint(0, 2 ** bits, (B, H * W), device="cuda", generator=g)
        ids[0, 0] = 1 << (bits - 1)  # MSB first: only channel 0 is +1
        Z = torch.full((B * (H + 2) * (W + 2), Cpad), SENT, device="cuda")
        call("mmdp_testing_lfq_to_padded", p(ids), p(Z), B, H, W, bits, Cpad)
        want = lfq_codebook_entry(ids.cpu(), bits).view(B, bits, H, W).permute(0, 2, 3, 1).cuda()
        zi = interior(Z, B, H, W)
        assert torch.equal(zi[..., :bits], want)
        assert zi[0, 0, 0, 0] == 1 and (zi[0, 0, 0, 1:bits] == -1).all()
        assert (zi[..., bits:] == SENT).all() and (Z[border_mask(B, H, W, Z.device)] == SENT).all()
        back = torch.full_like(ids, -1)
        call("mmdp_testing_lfq_indices", p(Z), p(back), B, H, W, bits, Cpad)
        assert torch.equal(back, ids)


@gpu
def test_codebook_to_padded():
    g = torch.Generator(device="cuda").manual_seed(5)
    for Cc, Cpad, n_codes, B, h, w in ((64, 64, 8192, 2, 16, 16), (16, 32, 512, 1, 3, 5), (13, 32, 1, 1, 1, 1)):
        cb = torch.randn(n_codes, Cc, device="cuda", generator=g)
        ids = torch.randint(0, n_codes, (B, h * w), device="cuda", generator=g)
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        Z = torch.full((B * (h + 2) * (w + 2), Cpad), SENT, device="cuda")
        call("mmdp_testing_codebook_to_padded", p(ids), p(cb), p(Z), B, h, w, Cc, Cpad, n_codes, p(err))
        zi = interior(Z, B, h, w)
        assert torch.equal(zi[..., :Cc], cb[ids].view(B, h, w, Cc)) and int(err) == 0
        assert (zi[..., Cc:] == SENT).all() and (Z[border_mask(B, h, w, Z.device)] == SENT).all()
        bad = ids.clone()
        bad[0, 0], bad[-1, -1] = -1, n_codes
        call("mmdp_testing_codebook_to_padded", p(bad), p(cb), p(Z), B, h, w, Cc, Cpad, n_codes, p(err))
        zi = interior(Z, B, h, w)
        assert int(err) & 1
        assert (zi[0, 0, 0, :Cc] == 0).all() and (zi[-1, -1, -1, :Cc] == 0).all()
        ok = torch.ones(B, h * w, dtype=torch.bool, device="cuda")
        ok[0, 0], ok[-1, -1] = False, False
        assert torch.equal(zi[..., :Cc].reshape(B, h * w, Cc)[ok], cb[ids][ok])


@gpu
@pytest.mark.parametrize("n", [1, 31, 256, 1024, 4096])
def test_softmax_rows_vs_fp64(n):
    g = torch.Generator(device="cuda").manual_seed(n)
    rows, ld = 37, r32(n) + 32
    s = torch.randn(rows, n, device="cuda", generator=g) * 4
    s[1] *= 30  # score range far over 80: terms underflow
    s[2, : max(1, n // 2)] -= 90
    s[3] = 5.0  # constant row
    buf = torch.full((rows, ld), SENT, device="cuda")
    buf[:, :n] = s
    call("mmdp_testing_softmax_rows_ld", p(buf), rows, n, ld)
    sd = s.double()
    ref = torch.softmax(sd, dim=-1)
    tol = ref * 2.0 ** -24 * ((sd - sd.amax(-1, keepdim=True)).abs() + n / 256 + 16) + 2.0 ** -126
    err = (buf[:, :n].double() - ref).abs()
    print(f"[softmax n={n}] max err {float(err.max()):.3e}, max err/bound {float((err / tol).max()):.3e}")
    assert (err <= tol).all()
    assert (buf[:, n:] == SENT).all()


# ------------------------------------------------------------------------------------------------------------------
# mmdp_vq_nearest
# ------------------------------------------------------------------------------------------------------------------
def vq_nearest(z, cb):
    from mmada_parallel_b200 import _lib
    B, Cc, h, w = z.shape
    ids = torch.empty(B * h * w, dtype=torch.int64, device=z.device)
    zq = torch.full_like(z, float("nan"))
    _lib.check(_lib.lib.mmdp_vq_nearest(p(z), p(cb), B, Cc, h, w, cb.shape[0], p(ids), p(zq), _lib.stream_ptr()))
    return ids, zq


def check_nearest(z, cb, ids, zq):
    """ids equal the fp64 argmin where the best-to-second gap exceeds tol = 1e-5 (|z|^2 + max|e|^2) (test_gpu_vqmodel.py),
    are within tol of the minimum everywhere, and zq is the chosen codebook rows bit for bit."""
    B, Cc, h, w = z.shape
    zr = z.permute(0, 2, 3, 1).reshape(-1, Cc).double()
    d = torch.cdist(zr, cb.double()) ** 2
    best = d.min(1)
    tol = 1e-5 * ((zr ** 2).sum(1) + (cb.double() ** 2).sum(1).max())
    if cb.shape[0] > 1:
        top2 = d.topk(2, largest=False).values
        decided = (top2[:, 1] - top2[:, 0]) > tol
    else:
        decided = torch.ones_like(ids, dtype=torch.bool)
    assert torch.equal(ids[decided], best.indices[decided])
    assert (d.gather(1, ids[:, None])[:, 0] - best.values <= tol).all()
    assert torch.equal(zq, cb[ids].view(B, h, w, Cc).permute(0, 3, 1, 2))
    return int(decided.sum())


@gpu
@pytest.mark.parametrize("C_", [1, 13, 64, 255, 256])
def test_vq_nearest_vs_fp64(C_):
    g = torch.Generator(device="cuda").manual_seed(C_)
    for n_codes in (1, 63, 64, 65, 4097, 8192):
        cb = torch.randn(n_codes, C_, device="cuda", generator=g)
        for B, h, w in ((1, 1, 1), (1, 1, 31), (1, 1, 33), (3, 24, 40)):
            z = torch.randn(B, C_, h, w, device="cuda", generator=g)
            ids, zq = vq_nearest(z, cb)
            decided = check_nearest(z, cb, ids, zq)
            if n_codes == 8192 and B == 3:
                print(f"[vq_nearest C={C_} codes={n_codes} N={B * h * w}] decided {decided}/{ids.numel()}")


@gpu
def test_vq_nearest_ties_and_exact_hits():
    """Duplicates of the winning code in different code-range splits (small N splits the codebook over ~2 CTAs per SM): the
    lowest index wins. A latent equal to a code has distance 0."""
    g = torch.Generator(device="cuda").manual_seed(9)
    for C_, n_codes, N in ((64, 8192, 1), (64, 8192, 31), (13, 4097, 33), (256, 8192, 2)):
        cb = torch.randn(n_codes, C_, device="cuda", generator=g)
        lo, hi = 5, n_codes - 3
        cb[hi] = cb[lo]
        z = cb[lo].view(1, C_, 1, 1).repeat(1, 1, 1, N) + 1e-3 * torch.randn(1, C_, 1, N, device="cuda", generator=g)
        z[0, :, 0, 0] = cb[lo]  # exact hit on a duplicated code
        if N > 1:
            z[0, :, 0, 1] = cb[77]  # exact hit on a unique code
        ids, zq = vq_nearest(z.contiguous(), cb)
        assert int(ids[0]) == lo and (N == 1 or int(ids[1]) == 77)
        assert (ids[2:] == lo).all(), "the lowest index must win a tie across code splits"
        assert torch.equal(zq, cb[ids].view(1, 1, N, C_).permute(0, 3, 1, 2))


@gpu
def test_vq_nearest_rejects_bad_channels():
    from mmada_parallel_b200 import _lib
    cb = torch.randn(64, 257, device="cuda")
    z = torch.randn(1, 257, 2, 2, device="cuda")
    ids = torch.empty(4, dtype=torch.int64, device="cuda")
    for Cc in (0, 257):
        assert _lib.lib.mmdp_vq_nearest(p(z), p(cb), 1, Cc, 2, 2, 64, p(ids), None, _lib.stream_ptr()) == -1
        assert b"C must be in [1, 256]" in _lib.lib.mmdp_last_error()


# ------------------------------------------------------------------------------------------------------------------
# two devices in one process
# ------------------------------------------------------------------------------------------------------------------
@gpu
def test_two_devices_bit_identical():
    """The tokenizers on cuda:1 after cuda:0 in one process: every launcher sets its shared-memory attribute per device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    from helpers import load_golden
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.magvit import MAGVITv2
    from mmada_parallel_b200.vqmodel import VQModel
    from oracle import amused as AM
    from oracle import magvit as OM
    gold = load_golden("amused_vq.pt")["small_attn"]
    acfg = AM.make_config(**gold["cfg"])
    aw = AM.make_weights(acfg, gold["weight_seed"])
    kw = dict(AM.AMUSED_CONFIG, **gold["cfg"])
    L = len(acfg.block_out_channels)
    kw.update(down_block_types=("DownEncoderBlock2D",) * L, up_block_types=("UpDecoderBlock2D",) * L, lookup_from_codebook=True)
    mcfg = OM.decoder_config(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 2))
    mw = OM.make_weights(mcfg, 1)
    aids = torch.randint(0, acfg.num_vq_embeddings, (1, 8, 8), generator=torch.Generator().manual_seed(0))
    mids = torch.randint(0, 8192, (1, 64), generator=torch.Generator().manual_seed(1))
    z = torch.randn(3, 64, 24, 40, generator=torch.Generator().manual_seed(2))
    cb = torch.randn(8192, 64, generator=torch.Generator().manual_seed(3))
    outs = []
    try:
        for dev in ("cuda:0", "cuda:1"):
            vm = VQModel(**kw, max_latent_cells=64, device=dev)
            vm.load_state_dict(aw)
            a = vm.decode(aids.to(dev), force_not_quantize=True, shape=(1, 8, 8, acfg.latent_channels)).sample
            mg = MAGVITv2(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 2), latent_hw=(8, 8), device=dev)
            mg.load_state_dict(mw)
            m = mg.decode_code(mids.to(dev))
            with torch.cuda.device(dev):
                zd, cbd = z.to(dev), cb.to(dev)
                ids = torch.empty(z.numel() // 64, dtype=torch.int64, device=dev)
                _lib.check(_lib.lib.mmdp_vq_nearest(p(zd), p(cbd), 3, 64, 24, 40, 8192, p(ids), None, _lib.stream_ptr()))
                torch.cuda.synchronize(dev)
            outs.append((a.cpu(), m.cpu(), ids.cpu()))
    finally:
        torch.cuda.set_device(0)
    for x, y in zip(*outs):
        assert torch.isfinite(x.double()).all() and torch.equal(x, y)
