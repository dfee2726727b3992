"""The QKV staged epilogue's rotary items (one item per row and 8-column group, spanning both heads of a tile and sharing their
cos / sin) and the last tile of each CTA, which the MMA warps drain together with the epilogue warps. Each launch is compared
bit for bit with the CTA-pair kernel, whose fused epilogue runs on the register fragments; both accumulate K in the same
order without the split-K tail. Covered: multi-head launches whose sequence boundaries fall inside 8-row groups, packed
batches (multi-head and grouped-query) with such boundaries, grouped-query and multi-query launches with a q / k / v bias
(MQA at 32 heads: one 256-wide tile ends k and starts V), and the attn_out residual launch in place."""
import contextlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def bf(x):
    return x.to(torch.bfloat16)


@contextlib.contextmanager
def kernel(pair):
    from mmada_parallel_b200 import _lib
    _lib.lib.mmdp_set_gemm_splitk(0)
    _lib.lib.mmdp_set_gemm_pair(1 if pair else 0)
    try:
        yield
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.lib.mmdp_set_gemm_pair(0)


def staged_and_register(fn):
    out = []
    for pair in (False, True):
        with kernel(pair):
            out.append([t.clone() for t in fn()])
    torch.cuda.synchronize()
    return out


def assert_same(got, ref, what):
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape, (what, i)
        assert torch.equal(g, r), f"{what}[{i}]: {int((g != r).sum())} of {g.numel()} elements differ"


def rope(L):
    from mmada_parallel_b200.model import rope_tables
    return [t.cuda() for t in rope_tables(128, 500000.0, L)]


@pytest.mark.parametrize("B,L,H", [(1, 2414, 32), (3, 333, 4), (2, 1001, 2)])
def test_qkv_rope(B, L, H):
    from mmada_parallel_b200 import _lib
    torch.manual_seed(B * L + H)
    d = 128 * H
    a = bf(torch.randn(B * L, d, device="cuda") * 0.5)
    w = bf(torch.randn(3 * d, d, device="cuda") / math.sqrt(d))
    cos, sin = rope(L)
    staged, reg = staged_and_register(lambda: _lib.qkv_rope(a, w, H, L, cos, sin))
    assert_same(staged, reg, f"qkv B={B} L={L} H={H}")
    assert staged[2].abs().sum() > 0


@pytest.mark.parametrize("H,Hkv,L", [(32, 8, 2414), (32, 1, 2414), (4, 2, 333)])
def test_qkv_gqa_bias(H, Hkv, L):
    from mmada_parallel_b200 import _lib
    torch.manual_seed(H * 100 + Hkv)
    d = 128 * H
    N = d + 2 * 128 * Hkv
    a = bf(torch.randn(L, d, device="cuda") * 0.5)
    w = bf(torch.randn(N, d, device="cuda") / math.sqrt(d))
    bias = bf(torch.randn(N, device="cuda") * 0.1)
    cos, sin = rope(L)
    staged, reg = staged_and_register(lambda: _lib.qkv_rope_gqa(a, w, bias, H, Hkv, L, cos, sin))
    assert_same(staged, reg, f"gqa H={H} Hkv={Hkv}")


@pytest.mark.parametrize("H,Hkv,bias", [(4, 4, False), (4, 2, True), (4, 1, True)])
def test_qkv_packed(H, Hkv, bias):
    """Sequences of 301, 77, 515 and 9 rows end to end: every boundary falls inside an 8-row group and inside a 128-row tile."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(H + 10 * Hkv)
    lens = [301, 77, 515, 9]
    M, d, dkv = sum(lens), 128 * H, 128 * Hkv
    N = d + 2 * dkv
    Lpad = (max(lens) + 7) // 8 * 8
    a = bf(torch.randn(M, d, device="cuda") * 0.5)
    w = bf(torch.randn(N, d, device="cuda") / math.sqrt(d))
    b = bf(torch.randn(N, device="cuda") * 0.1) if bias else None
    cos, sin = rope(Lpad)
    seg = torch.tensor(lens, dtype=torch.int32)
    row_map = torch.empty(M, 2, dtype=torch.int32, device="cuda")

    def run():
        q = torch.empty(M, d, dtype=torch.bfloat16, device="cuda")
        k = torch.empty(M, dkv, dtype=torch.bfloat16, device="cuda")
        vt = torch.zeros(len(lens), Hkv, 128, Lpad, dtype=torch.bfloat16, device="cuda")
        _lib.check(_lib.lib.mmdp_qkv_rope_tp_packed(_lib.PRECISION_BF16, _lib.ptr(a), d, None, _lib.ptr(w), None, _lib.ptr(b), d, H,
                                                    Hkv, len(lens), seg.data_ptr(), Lpad, _lib.ptr(cos), _lib.ptr(sin), _lib.ptr(q),
                                                    _lib.ptr(k), _lib.ptr(vt), _lib.ptr(row_map), _lib.stream_ptr()))
        return q, k, vt

    staged, reg = staged_and_register(run)
    assert_same(staged, reg, f"packed H={H} Hkv={Hkv} bias={bias}")
    assert staged[2].abs().sum() > 0


def test_residual_in_place():
    """attn_out + residual at the production shape: 304 tiles, so every CTA's last tile is drained by all of its warps."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(7)
    M, N, K = 2414, 4096, 4096
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.02)
    r0 = bf(torch.randn(M, N, device="cuda"))

    def run():
        r = r0.clone()
        _lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r, out=r)
        return (r,)

    staged, reg = staged_and_register(run)
    assert_same(staged, reg, "resid in place")
    assert not torch.equal(staged[0], r0)
