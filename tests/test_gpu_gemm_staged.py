"""The staged epilogue of gemm_bf16_kernel (the MMA warps hand each tile to the epilogue warps as bf16 through shared memory)
against the CTA-pair kernel, which keeps the fused epilogue on the register fragments. Every epilogue rounds the accumulator
to bf16 before anything else and both kernels accumulate K in the same order without the split-K tail, so the outputs must
agree bit for bit: QKV + RoPE (q, k and V^T), residual in place, plain, SwiGLU, partial tiles, a 192-wide tile plan, a grid
smaller than the SM count, and whole forwards of the tiny model in the ordinary, token-cache and packed modes."""
import contextlib
import math

import pytest
import torch

from helpers import load_golden, tiny_cfg_and_weights

pytestmark = pytest.mark.gpu


def bf(x):
    return x.to(torch.bfloat16)


@contextlib.contextmanager
def kernel(pair):
    """Split-K tail off (the pair kernel has none); pair = 1 selects the CTA-pair kernel for every launch with M > 256."""
    from mmada_parallel_b200 import _lib
    _lib.lib.mmdp_set_gemm_splitk(0)
    _lib.lib.mmdp_set_gemm_pair(1 if pair else 0)
    try:
        yield
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.lib.mmdp_set_gemm_pair(0)


def both(fn):
    """fn() under the staged (default) kernel and under the pair kernel; every returned tensor is cloned."""
    out = []
    for pair in (False, True):
        with kernel(pair):
            r = fn()
        out.append([t.clone() for t in (r if isinstance(r, (tuple, list)) else (r,))])
    torch.cuda.synchronize()
    return out


def assert_same(got, ref, what):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape, (what, i)
        if not torch.equal(g, r):
            n = int((g != r).sum())
            raise AssertionError(f"{what}[{i}]: {n} of {g.numel()} elements differ")


@pytest.mark.parametrize("B,L,H", [(1, 2414, 32), (3, 333, 4), (2, 1001, 2)])
def test_qkv_rope_bit_identical(B, L, H):
    """Production QKV (2414 x 12288 x 4096), and batches whose sequence boundaries fall inside 8-row groups (L % 8 != 0), so
    that V^T takes both its 16-byte and its element stores."""
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import rope_tables
    torch.manual_seed(L + H)
    d = 128 * H
    a = bf(torch.randn(B * L, d, device="cuda") * 0.5)
    w = bf(torch.randn(3 * d, d, device="cuda") / math.sqrt(d))
    cos, sin = (t.cuda() for t in rope_tables(128, 500000.0, L))
    staged, pair = both(lambda: _lib.qkv_rope(a, w, H, L, cos, sin))
    assert_same(staged, pair, f"qkv B={B} L={L}")
    assert staged[2].abs().sum() > 0


@pytest.mark.parametrize("M,N,K", [(2414, 4096, 4096), (333, 1000, 520), (384, 512, 256)])
def test_residual_in_place_bit_identical(M, N, K):
    """C is the residual (the forward's x += attn_out / ff_out), M % 128 != 0, N % 256 != 0, and 6 tiles (< 132 SMs)."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M + N)
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    r0 = bf(torch.randn(M, N, device="cuda"))

    def run():
        r = r0.clone()
        out = _lib.gemm_bf16(a, w, _lib.EPI_RESID, resid=r, out=r)
        assert out.data_ptr() == r.data_ptr()
        return r

    staged, pair = both(run)
    assert_same(staged, pair, "resid in place")
    assert not torch.equal(staged[0], r0)


@pytest.mark.parametrize("M,N,K", [(333, 1000, 520), (2414, 2304, 512), (384, 768, 1024)])
def test_plain_bit_identical(M, N, K):
    """N % 256 != 0; 2414 x 2304 is planned with 192-wide tiles (228 tiles: 2 waves, against 171 tiles of 256, also 2 waves);
    384 x 768 is 9 tiles on 132 SMs."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M * 3 + N)
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.05)
    staged, pair = both(lambda: _lib.gemm_bf16(a, w, _lib.EPI_PLAIN))
    assert_same(staged, pair, "plain")
    ref = bf(a.float() @ w.float().t()).float()
    assert (staged[0].float() - ref).abs().max() <= 2.0 ** -7 * ref.abs().max()


@pytest.mark.parametrize("M", [2414, 300])
def test_swiglu_bit_identical(M):
    """The gate/up production shape: 1824 tiles, about 14 per CTA through the same staging tile."""
    from mmada_parallel_b200 import _lib
    torch.manual_seed(M)
    K, N = 4096, 24576
    a = bf(torch.randn(M, K, device="cuda") * 0.5)
    w = bf(torch.randn(N, K, device="cuda") * 0.02)
    staged, pair = both(lambda: _lib.gemm_bf16(a, w, _lib.EPI_SWIGLU))
    assert_same(staged, pair, "swiglu")


def _tiny(max_batch=4):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    meta = load_golden("trajectory_a_tiny.pt")["meta"]
    cfg, sd = tiny_cfg_and_weights(meta)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=max_batch)
    m.load_state_dict(sd)
    return m


def _ids(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 134656, shape, generator=g).cuda()


def test_forward_ordinary_bit_identical():
    """Whole forwards (every block GEMM, the head) with one and with two sequences (L = 301: boundaries inside 8-row groups)."""
    m = _tiny()
    for ids in (_ids((1, 500), 1), _ids((2, 301), 2)):
        staged, pair = both(lambda: m(ids, infer=True, use_cache=False).logits)
        assert_same(staged, pair, f"forward {tuple(ids.shape)}")
    m.raise_device_errors()


def test_forward_token_cache_bit_identical():
    """Token-cache forward: the partial recompute runs QKV with a position map (k rows and V^T columns scattered into the
    cache at their positions, which are not consecutive)."""
    m = _tiny()
    ids = _ids((1, 500), 3)
    g = torch.Generator().manual_seed(4)
    mask = torch.rand(1, 500, generator=g) < 0.55
    mask[0, 100:180] = True  # one run of consecutive positions as well
    ids2 = ids.clone()
    ids2[mask.cuda()] = 126336

    def run():
        m.caching(True)
        try:
            m(ids, infer=True, use_cache=True, cat="k")
            out = m(ids2, infer=True, use_cache=True, to_compute_mask=mask, cat="k").logits.clone()
            m.empty_cache()
        finally:
            m.caching(False)
        return out

    assert int(mask.sum()) > 256  # the pair kernel serves launches with M > 256
    staged, pair = both(run)
    assert_same(staged, pair, "token-cache forward")
    m.raise_device_errors()


def test_forward_packed_bit_identical():
    """Packed forward of four sequences: per-row (sequence, position) map, boundaries inside 8-row groups."""
    m = _tiny()
    lens = [300, 77, 512, 129]
    ids = _ids((sum(lens),), 5)
    rows_a = torch.arange(0, sum(lens), 3, dtype=torch.int32, device="cuda")
    rows_b = torch.arange(1, sum(lens), 4, dtype=torch.int32, device="cuda")
    staged, pair = both(lambda: m.forward_rows_packed(ids, lens, rows_a=rows_a, rows_b=rows_b, col0_b=126356, ncols_b=8192))
    assert_same(staged, pair, "packed forward")
    m.raise_device_errors()
