"""CPU self-test of the comparators in tp_ops_ref.py that tests/test_gpu_tp_ops.py applies to the tensor-parallel kernels: each
accepts the exact emulation of its kernel and rejects a result that is subtly wrong in the way a kernel bug would make it
(one bf16 ulp, the wrong summation order, a missing rounding point, eps in the wrong place, a row in the neighbour's buffer).
This is what makes the GPU tests fail when a kernel is wrong."""
import pytest
import torch

from tp_ops_ref import (GEMM_MEAN_FRAC, bf16r, bits, bitwise_mismatch, emulate_reduce, emulate_resid_add, gemm_f32_reference, gemm_f32_violations,
                        is_sentinel, norm_inputs, norm_mismatch, owned_rows, reduce_partials, resid_inputs, scatter_expected,
                        scatter_mismatch, sentinel_f32)


def _gemm_case(M=40, N=36, K=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    return a, w


def test_gemm_bound_accepts_fp32_accumulation():
    a, w = _gemm_case()
    ref, bound = gemm_f32_reference(a, w)
    # a sequential fp32 sum (the worst accumulation order) and torch's fp32 matmul are both inside
    seq = torch.zeros(a.shape[0], w.shape[0])
    af, wf = a.float(), w.float()
    for k in range(a.shape[1]):
        seq = seq + af[:, k:k + 1] * wf[:, k][None, :]
    for got in (seq, af @ wf.t()):
        mx, mean = gemm_f32_violations(got, ref, bound)
        assert mx <= 1.0 and mean <= GEMM_MEAN_FRAC, (mx, mean)


def test_gemm_bound_rejects_dropped_kblock_and_wrong_column():
    a, w = _gemm_case()
    ref, bound = gemm_f32_reference(a, w)
    af, wf = a.float(), w.float()
    dropped = af[:, 64:] @ wf[:, 64:].t()                   # one 64-deep k-block missing
    shifted = (af @ wf.t())[:, [1, 0] + list(range(2, w.shape[0]))]   # two columns exchanged
    one = (af @ wf.t()).clone()
    one[3, 5] = float(ref[3, 5]) + 50 * float(bound[3, 5])  # a single element far off
    for bad in (dropped, shifted, one):
        mx, mean = gemm_f32_violations(bad, ref, bound)
        assert mx > 1.0
    assert gemm_f32_violations(dropped, ref, bound)[1] > 100 * GEMM_MEAN_FRAC   # by orders of magnitude
    assert gemm_f32_violations(torch.full_like(ref, float("nan")).float(), ref, bound)[0] > 1.0


@pytest.mark.parametrize("M,n", [(2414, 8), (9, 4), (335, 3)])
def test_scatter_expectation_rejects_misplaced_rows(M, n):
    N = 12
    R = (M + n - 1) // n
    rows = torch.randn(M, N)
    slot = n - 1
    want = scatter_expected(rows, n, R, slot)
    assert scatter_mismatch([t.clone() for t in want], want) is None
    # every row where it belongs, the rest sentinel
    for r in range(n):
        row0, nrows = owned_rows(M, n, r)
        assert torch.equal(bits(want[r][slot, :nrows]), bits(rows[row0:row0 + nrows]))
        assert is_sentinel(want[r][slot, nrows:]) and is_sentinel(want[r][:slot])
    if M == 9:
        assert is_sentinel(want[3]), "the last rank owns no row: its buffer stays untouched"
    # a row written to the neighbouring owner, to the neighbouring slot, or one row off
    last = M - 1
    o, i = last // R, last % R
    bad_owner = [t.clone() for t in want]
    bad_owner[o - 1][slot, i] = rows[last]
    bad_slot = [t.clone() for t in want]
    bad_slot[o][slot - 1 if slot else 1, i] = rows[last]
    bad_slot[o][slot, i] = sentinel_f32(N)
    off_by_one = [t.clone() for t in want]
    off_by_one[0][slot, 1:R] = rows[0:R - 1]
    for bad in (bad_owner, bad_slot, off_by_one):
        assert scatter_mismatch(bad, want) is not None


def test_resid_add_emulation_pins_both_roundings():
    x, p = resid_inputs(4, 1000, seed=1)
    want = emulate_resid_add(x, p)
    assert bitwise_mismatch(emulate_resid_add(x, p), want) == 0
    wb = bits(want)
    # the edge cases are present: exact +0 and -0, +-inf, bf16 subnormals
    assert bool((wb == 0).any()) and bool((wb == torch.tensor(-32768, dtype=torch.int16)).any())
    assert bool(torch.isinf(want.float()).any())
    sub = (want.float() != 0) & (want.float().abs() < 2.0 ** -126)
    assert bool(sub.any())
    # a missing rounding point of the partial, or a partial rounded toward zero instead of to nearest, is rejected
    no_inner = (x.float() + p).to(torch.bfloat16)
    trunc = (x.float() + (p.view(torch.int32) & ~0xFFFF).view(torch.float32)).to(torch.bfloat16)
    for bad in (no_inner, trunc):
        assert bitwise_mismatch(bad, want) > 0
    # a result one ulp off in a single ordinary element is rejected, and counted as exactly one element
    finite = torch.isfinite(want.float()) & (want.float().abs() >= 2.0 ** -126)
    i = int(finite.view(-1).nonzero()[0])
    flip = wb.clone().view(-1)
    flip[i] += 1
    assert bitwise_mismatch(flip.view(want.shape).view(torch.bfloat16), want) == 1


@pytest.mark.parametrize("n", [4, 8])
def test_reduce_emulation_pins_rank_order(n):
    parts = reduce_partials(n, 16, 256, seed=n)
    x = (torch.randn(16, 256) * 2).to(torch.bfloat16)
    want = emulate_reduce(parts, x)
    rev = emulate_reduce(parts, x, order=list(reversed(range(n))))
    rot = emulate_reduce(parts, x, order=list(range(1, n)) + [0])
    assert bitwise_mismatch(rev, want) > 0.05 * want.numel(), "the inputs must make the summation order visible"
    assert bitwise_mismatch(rot, want) > 0.05 * want.numel()
    # a missing bf16 rounding of the sum is rejected too
    s = torch.zeros_like(parts[0])
    for t in parts:
        s = s + t
    assert bitwise_mismatch((x.float() + s).to(torch.bfloat16), want) > 0


def test_reduce_two_ranks_order_is_commutative():
    """With two sources the sum (0 + p0) + p1 is one fp32 add, which is commutative: no order to pin at n = 2."""
    parts = reduce_partials(2, 8, 64, seed=5)
    x = torch.zeros(8, 64, dtype=torch.bfloat16)
    assert bitwise_mismatch(emulate_reduce(parts, x, order=[1, 0]), emulate_reduce(parts, x)) == 0


def _norm_variants(x, w, eps):
    xf = x.float()
    d = x.shape[1]
    ms = xf.pow(2).mean(-1, keepdim=True)
    wf = w.float()
    good = torch.rsqrt(ms + eps)
    return {
        "fp32 rstd (a different but legitimate fp32 evaluation)": (wf * bf16r(xf * (1.0 / torch.sqrt(ms + eps)))).to(torch.bfloat16),
        "eps added after the sqrt": (wf * bf16r(xf / (torch.sqrt(ms) + eps))).to(torch.bfloat16),
        "no eps": (wf * bf16r(xf / torch.sqrt(ms))).to(torch.bfloat16),
        "divisor d + 8": (wf * bf16r(xf * torch.rsqrt(xf.pow(2).sum(-1, keepdim=True) / (d + 8) + eps))).to(torch.bfloat16),
        "missing bf16 rounding of x * rstd": (wf * (xf * good)).to(torch.bfloat16),
        "weight applied before the rounding": bf16r(wf * xf * good).to(torch.bfloat16),
    }


@pytest.mark.parametrize("d", [256, 1000, 4096])
def test_norm_check_boundary_aware(d):
    eps = 1e-5
    x, w = norm_inputs(64, d, seed=d)
    variants = _norm_variants(x, w, eps)
    bad, ties = norm_mismatch(variants.pop("fp32 rstd (a different but legitimate fp32 evaluation)"), x, w, eps)
    assert bad == 0 and ties <= 0.02 * x.numel(), (bad, ties)
    for name, y in variants.items():
        bad, _ = norm_mismatch(y, x, w, eps)
        assert bad > 0.01 * x.numel() or (name == "eps added after the sqrt" and bad > 0), (name, bad)
    # one bf16 ulp flipped in a non-tie element
    from tp_ops_ref import norm_expected
    y_near, _, tie = norm_expected(x, w, eps)
    idx = int((~tie & (y_near.float() != 0)).view(-1).nonzero()[0])
    flipped = bits(y_near).clone().view(-1)
    flipped[idx] += 1
    assert norm_mismatch(flipped.view(x.shape).view(torch.bfloat16), x, w, eps)[0] == 1
