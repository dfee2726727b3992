"""Reference emulations and comparators of the tensor-parallel kernels: the fp32 GEMM output (MMDP_EPI_F32) and its scatter into
the owners' receive buffers, mmdp_resid_add_f32, mmdp_tp_reduce_norm (csrc/tp_collective.cu) and mmdp_rmsnorm.

Plain torch, device agnostic: tests/test_gpu_tp_ops.py runs them next to the kernels on the GPU, tests/test_tp_ops_host.py
shows on the CPU that each comparator accepts the exact emulation and rejects a subtly wrong result. torch's float32 adds and
its float32 -> bfloat16 conversion round to nearest even on both devices, so the emulations are exact.
"""
from __future__ import annotations

import math

import torch

# GEMM bound: |C - A W^T| <= GEMM_C * K * 2^-24 * (|A| |W|^T) per element. The classic bound of a K-term fp32 sum is
# K * 2^-24 * sum |a w|; GEMM_C = 2 leaves room for an accumulator that truncates instead of rounding (unit 2^-23).
GEMM_C = 2.0
# ... and on average the error sits orders of magnitude inside it (random rounding errors grow like sqrt(K), the bound like K).
GEMM_MEAN_FRAC = 1.0 / 64
# Norm check: an element whose exact n = x * rstd lies within this relative distance of a bf16 rounding midpoint may round
# either way. The kernel's fp32 rstd (a sum of <= 8192 squares in a tree of <= 40 levels, a divide, sqrt and reciprocal) is
# within ~2^-19 of the fp64 one, so 2^-16 is safe, yet it admits only ~1 % of the elements.
NORM_TIE_REL = 2.0 ** -16

SENTINEL_F32 = 0x7FC0DEAD  # int32 bits of an fp32 NaN no kernel produces
SENTINEL_BF16 = 0x7FA5     # int16 bits of a bf16 NaN


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """Round fp32 to bf16 (nearest even) and back."""
    return x.to(torch.bfloat16).float()


def bits(t: torch.Tensor) -> torch.Tensor:
    """Integer view of a float tensor, so that comparisons are bitwise (NaN payloads, the sign of zero)."""
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16}[t.dtype])


def bitwise_mismatch(got: torch.Tensor, want: torch.Tensor) -> int:
    """Number of elements whose bits differ: the comparator of every result that must be exact."""
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    return int((bits(got) != bits(want.to(got.device))).sum())


def sentinel_f32(*shape, device="cpu") -> torch.Tensor:
    return torch.full(shape, SENTINEL_F32, dtype=torch.int32, device=device).view(torch.float32)


def sentinel_bf16(*shape, device="cpu") -> torch.Tensor:
    return torch.full(shape, SENTINEL_BF16, dtype=torch.int16, device=device).view(torch.bfloat16)


def is_sentinel(t: torch.Tensor) -> bool:
    return bool((bits(t) == (SENTINEL_F32 if t.dtype == torch.float32 else SENTINEL_BF16)).all())


# ---- fp32 GEMM -----------------------------------------------------------------------------------------------------------
def gemm_f32_reference(a: torch.Tensor, w: torch.Tensor):
    """fp64 A W^T and the per-element bound GEMM_C * K * 2^-24 * (|A| |W|^T)."""
    a64, w64 = a.double(), w.double()
    ref = a64 @ w64.t()
    bound = GEMM_C * a.shape[1] * 2.0 ** -24 * (a64.abs() @ w64.abs().t())
    return ref, bound


def gemm_f32_violations(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor):
    """(max, mean) of |got - ref| / bound; a result passes with max <= 1 and mean <= GEMM_MEAN_FRAC."""
    g = got.double()
    if not torch.isfinite(g).all():
        return math.inf, math.inf
    r = (g - ref).abs() / bound.clamp_min(1e-300)
    return r.max().item(), r.mean().item()


def assert_gemm_f32(got, ref, bound, what):
    mx, mean = gemm_f32_violations(got, ref, bound)
    assert mx <= 1.0, f"{what}: error {mx:.3g} x the bound {GEMM_C} K 2^-24 |A||W|^T"
    assert mean <= GEMM_MEAN_FRAC, f"{what}: mean error {mean:.3g} x the bound (must stay below {GEMM_MEAN_FRAC})"


# ---- scatter of fp32 rows to their owners ---------------------------------------------------------------------------------
def owned_rows(M: int, n: int, r: int):
    """Rows [row0, row0 + nrows) that rank r owns: R = ceil(M / n), owner of a row = row // R."""
    R = (M + n - 1) // n
    row0 = r * R
    return row0, max(0, min(R, M - row0))


def scatter_expected(rows: torch.Tensor, n: int, R: int, slot: int):
    """The receive buffers ([n][R][N] fp32 each, pre-filled with the sentinel) after rank `slot` pushed every row of `rows`
    [M, N] to recv[row // R][slot][row % R]."""
    M, N = rows.shape
    out = [sentinel_f32(n, R, N, device=rows.device) for _ in range(n)]
    for r in range(n):
        lo, hi = r * R, min((r + 1) * R, M)
        if hi > lo:
            out[r][slot, :hi - lo] = rows[lo:hi]
    return out


def scatter_mismatch(got, want):
    """None when every receive buffer matches bit for bit, else a description of the first difference."""
    for r, (g, w) in enumerate(zip(got, want)):
        diff = bits(g) != bits(w)
        if diff.any():
            s, i, c = (int(v) for v in diff.nonzero()[0])
            return f"recv[{r}][slot {s}][row {i}][col {c}]: {int(diff.sum())} words differ"
    return None


# ---- residual add and the tensor-parallel reduce --------------------------------------------------------------------------
def emulate_resid_add(x: torch.Tensor, partial: torch.Tensor) -> torch.Tensor:
    """x = bf16(bf16(partial) + x): the rounding points of mmdp_resid_add_f32."""
    return (x.float() + bf16r(partial)).to(torch.bfloat16)


def resid_inputs(M: int, d: int, seed: int):
    """x bf16 [M, d] and fp32 partials [M, d] that exercise the rounding edges: partials that cancel x to +0 (and -0 + -0),
    values in and near the bf16 / fp32 subnormal range, sums that overflow bf16 to +-inf, partials that lie on or next to a
    bf16 rounding midpoint, and ordinary values."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, d, generator=g) * 4).to(torch.bfloat16)
    p = torch.randn(M, d, generator=g) * 4
    kind = torch.randint(0, 8, (M, d), generator=g)
    xf = x.float()
    p = torch.where(kind == 1, -xf, p)                                            # x + (-x) = +0
    sub = torch.randn(M, d, generator=g) * 2.0 ** -128                            # subnormal-ish partials (fp32 and bf16)
    p = torch.where(kind == 2, sub, p)
    x = torch.where(kind == 2, (torch.randn(M, d, generator=g) * 2.0 ** -127).to(torch.bfloat16), x)
    big = torch.finfo(torch.bfloat16).max
    p = torch.where(kind == 3, torch.sign(xf + 0.5) * big, p)                     # overflows bf16 when added to x of the same sign
    x = torch.where(kind == 3, (torch.sign(xf + 0.5) * big).to(torch.bfloat16), x)
    # a bf16 value plus half its spacing (a tie: rounds to even), plus a little more (rounds up) - inner rounding matters
    b = bf16r(p)
    half = b.abs() * 2.0 ** -8
    p = torch.where(kind == 4, b + half, p)
    p = torch.where(kind == 5, b + half * 1.0001, p)
    x = torch.where(kind == 6, torch.full_like(x, -0.0), x)
    p = torch.where(kind == 6, torch.full_like(p, -0.0), p)                       # -0 + -0 = -0
    return x, p.float()


def reduce_partials(n: int, nrows: int, d: int, seed: int):
    """n fp32 partial-sum blocks [nrows, d] of mixed sign and magnitude, so that the fp32 summation order shows in the
    bf16-rounded sum: a quarter of the elements carry +-B on rank 0, -+B on rank 1 and small values elsewhere (the forward
    order cancels B first, another order loses the small values against B); the rest are ordinary values of varied scale."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, nrows, d, generator=g) * torch.exp2(torch.randint(-6, 4, (n, nrows, d), generator=g).float())
    if n >= 2:
        sel = torch.rand(nrows, d, generator=g) < 0.25
        B = torch.exp2(torch.randint(20, 30, (nrows, d), generator=g).float()) * torch.sign(torch.randn(nrows, d, generator=g))
        p[0] = torch.where(sel, B, p[0])
        p[1] = torch.where(sel, -B, p[1])
    return [p[r].contiguous() for r in range(n)]


def emulate_reduce(parts, x: torch.Tensor, order=None) -> torch.Tensor:
    """x = bf16(bf16(sum) + x) with sum = ((0 + p_0) + p_1) + ... in fp32, in rank order (or `order`)."""
    s = torch.zeros_like(parts[0])
    for r in (range(len(parts)) if order is None else order):
        s = s + parts[r]
    return (x.float() + bf16r(s)).to(torch.bfloat16)


# ---- RMSNorm: boundary-aware exact check ----------------------------------------------------------------------------------
def norm_expected(x: torch.Tensor, w: torch.Tensor, eps: float):
    """For y = bf16(w * bf16(x * rstd)) with rstd = 1 / sqrt(mean(x^2) + eps): the result from the fp64 rstd (y_near), the
    result from the other bf16 neighbour of n = x * rstd (y_alt) and the elements whose n lies within NORM_TIE_REL of a
    rounding midpoint (tie), where either is accepted. w * bf16(n) is exact in fp32, so y has one rounding of its own."""
    x64 = x.double()
    rstd = 1.0 / torch.sqrt(x64.pow(2).mean(-1, keepdim=True) + eps)
    n = x64 * rstd
    an = n.abs()
    e = torch.frexp(an.clamp_min(2.0 ** -126)).exponent.double() - 1     # an in [2^e, 2^(e+1)), exactly
    ulp = torch.exp2(e - 7)                                                # bf16 spacing there
    q = an / ulp
    fl = torch.floor(q)
    frac = q - fl
    sgn = torch.where(n < 0, -1.0, 1.0).double()
    lo, hi = sgn * fl * ulp, sgn * (fl + 1) * ulp
    zero = an == 0
    near = torch.where(zero, n, torch.where(frac < 0.5, lo, hi))
    alt = torch.where(zero, n, torch.where(frac < 0.5, hi, lo))
    tie = ~zero & ((frac - 0.5).abs() * ulp <= NORM_TIE_REL * an)
    wf = w.float()
    y_near = (wf * near.float()).to(torch.bfloat16)
    y_alt = (wf * alt.float()).to(torch.bfloat16)
    return y_near, y_alt, tie


def norm_mismatch(y: torch.Tensor, x: torch.Tensor, w: torch.Tensor, eps: float):
    """(number of elements that are neither the exact result nor, at a tie, the other neighbour's; number of ties)."""
    y_near, y_alt, tie = norm_expected(x, w, eps)
    yb = bits(y)
    ok = (yb == bits(y_near)) | (tie & (yb == bits(y_alt)))
    return int((~ok).sum()), int(tie.sum())


def assert_norm_exact(y, x, w, eps, what):
    bad, ties = norm_mismatch(y, x, w, eps)
    assert bad == 0, f"{what}: {bad} of {y.numel()} elements are not the correctly rounded bf16(w * bf16(x * rstd))"
    assert ties <= 0.02 * y.numel(), f"{what}: {ties} near-tie elements (the tolerance admits too many)"


def norm_inputs(M: int, d: int, seed: int):
    """bf16 rows whose scale varies from 1e-3 to 3 (mean squares from far below eps = 1e-5 to far above it, so eps matters
    in some rows) and a norm weight around 1. Returns (x [M, d], w [d])."""
    g = torch.Generator().manual_seed(seed)
    scale = torch.exp(torch.empty(M, 1).uniform_(math.log(1e-3), math.log(3.0), generator=g))
    x = (torch.randn(M, d, generator=g) * scale).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(d, generator=g)).to(torch.bfloat16)
    return x, w
