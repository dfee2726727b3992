"""The tensor-parallel kernels op by op on ONE GPU, against exact emulations or fp64 references (tp_ops_ref.py):

  EPI_F32 GEMM output            within 2 K 2^-24 (|A| |W|^T) of fp64 A W^T, mean error far inside; split-K tail repeatable
  mmdp_gemm_f32_scatter          every row bitwise at recv[row // R][slot][row % R], everything else keeps its sentinel
  mmdp_resid_add_f32             bitwise equal to (x + bf16(partial)) rounded to bf16
  mmdp_tp_reduce_norm            x_shard bitwise equal to the rank-order fp32 sum emulation; xn boundary-aware exact; the
                                 broadcast, the phase flags and the done counter
  mmdp_qkv_rope_tp               fp32 reference (ulp bounds) and bitwise equal to its heads' slice of mmdp_qkv_rope
  mmdp_tp_forward (1 rank)       oracle within 4 bf16 ulp; two row chunks bitwise equal to one; epoch arithmetic
  TP = 2 / 4 / 8 op by op        the per-layer sequence of mmdp_tp_forward on simulated ranks
  mmdp_rmsnorm                   boundary-aware exact on every dispatch branch

The kernels take device pointers only, so "every rank's buffer" is a separate allocation on the same device and the simulated
ranks run one after another on one stream. The flag waits of csrc/tp_collective.cu spin until a peer writes a flag (and trap
after 2^27 polls), so before each mmdp_tp_reduce_norm call of a simulated rank every flag that call waits on is set to the
call's epoch, on the same stream: no wait inside the call can spin. mmdp_tp_forward is only called with one rank, whose waits
are on flags it writes itself earlier in stream order."""
import ctypes as C
import math

import pytest
import torch

from tp_ops_ref import (assert_gemm_f32, assert_norm_exact, bits, bitwise_mismatch, emulate_reduce, emulate_resid_add,
                        gemm_f32_reference, is_sentinel, norm_inputs, owned_rows, reduce_partials, resid_inputs, scatter_expected,
                        scatter_mismatch, sentinel_bf16, sentinel_f32)

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _lib():
    from mmada_parallel_b200 import _lib
    return _lib


def _stream():
    return _lib().stream_ptr()


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class _Options:
    """GEMM switches for the duration of a test; the defaults (split-K mode 2, pair kernel off) are restored in any case."""

    def __init__(self, splitk=None, pair=None):
        self.splitk, self.pair = splitk, pair

    def __enter__(self):
        lib = _lib().lib
        if self.splitk is not None:
            lib.mmdp_set_gemm_splitk(self.splitk)
        if self.pair is not None:
            lib.mmdp_set_gemm_pair(self.pair)
        return self

    def __exit__(self, *exc):
        lib = _lib().lib
        lib.mmdp_set_gemm_splitk(2)
        lib.mmdp_set_gemm_pair(0)
        return False


def _rand_bf16(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def gemm_f32(a, w, ldc=None):
    """MMDP_EPI_F32: C [M, ldc] fp32 (columns >= N keep their sentinel)."""
    L = _lib()
    M, K = a.shape
    N = w.shape[0]
    c = sentinel_f32(M, ldc or N, device=DEV)
    L.check(L.lib.mmdp_gemm_bf16(L.EPI_F32, a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), M, N, K, c.data_ptr(),
                                 c.stride(0), None, 0, _stream()))
    return c


def plan_width(M, N, sms):
    """Tile width plan_gemm (csrc/gemm.cu) picks for an EPI_F32 launch with the split-K tail off: the restatement of
    tools/bench_gemm.py (waves_no_split), cost = waves x width, 192-wide tiles charged 4 % more."""
    best = None
    for bn in (256, 192):
        waves = -(-(-(-M // 128) * -(-N // bn)) // sms)
        cost = waves * bn * (1.04 if bn == 192 else 1.0)
        if best is None or cost < best[0]:
            best = (cost, bn)
    return best[1]


# ---------------------------------------------------------------------------------------------------------------------------
# 1. fp32 GEMM output and the fused scatter
# ---------------------------------------------------------------------------------------------------------------------------
F32_SHAPES = [  # (M, N, K, ldc)
    (300, 768, 512, None),      # 192-wide tiles win (one wave either way)
    (2414, 4096, 512, None),    # 256-wide tiles win (3 waves against 4)
    (333, 1020, 264, None),     # N % 8 == 4: the float2 column tail; ragged M
    (1, 1020, 256, None),       # a single row
    (129, 520, 128, 528),       # ldc > N
    (7, 8, 8, 12),              # the smallest problem, ldc > N
]
TP_BENCH_SHAPES = [(2414, 4096, k // tp) for tp in (2, 4, 8) for k in (4096, 12288)]


def test_f32_gemm_shapes_cover_both_tile_widths():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    widths = {plan_width(M, N, sms) for M, N, _, _ in F32_SHAPES}
    assert widths == {192, 256}, (sms, widths)


@pytest.mark.parametrize("M,N,K,ldc", F32_SHAPES + [(M, N, K, None) for M, N, K in TP_BENCH_SHAPES])
def test_gemm_f32_against_fp64(M, N, K, ldc):
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a = _rand_bf16(g, M, K, scale=0.5)
    w = _rand_bf16(g, N, K, scale=K ** -0.5)
    ref, bound = gemm_f32_reference(a, w)
    with _Options(splitk=0):
        c = gemm_f32(a, w, ldc)
    assert_gemm_f32(c[:, :N], ref, bound, f"EPI_F32 {M}x{N}x{K}")
    if ldc:
        assert is_sentinel(c[:, N:]), "columns past N of a row with ldc > N must stay untouched"


@pytest.mark.parametrize("M,N,K", [(300, 1020, 1024), (1, 1020, 512), (2414, 4096, 2048), (2414, 4096, 1536)])
def test_gemm_f32_splitk_tail(M, N, K):
    """Split-K mode 3 splits every partial last wave: the finishing pass (epi_row8's float4 stores, with the float4 tail at
    N % 8 == 4) stays inside the same bound and is bitwise repeatable."""
    g = torch.Generator().manual_seed(M + N + K)
    a = _rand_bf16(g, M, K, scale=0.5)
    w = _rand_bf16(g, N, K, scale=K ** -0.5)
    ref, bound = gemm_f32_reference(a, w)
    with _Options(splitk=3):
        c1 = gemm_f32(a, w)
        c2 = gemm_f32(a, w)
    assert_gemm_f32(c1, ref, bound, f"EPI_F32 split-K {M}x{N}x{K}")
    assert bitwise_mismatch(c1, c2) == 0, "the split-K tail must be deterministic"


def gemm_scatter(a, w, recv, R, slot):
    L = _lib()
    M, K = a.shape
    N = w.shape[0]
    L.check(L.lib.mmdp_gemm_f32_scatter(a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), M, N, K, _ptrs(recv), len(recv), R,
                                        slot, _stream()))


@pytest.mark.parametrize("M,N,K,n", [(335, 264, 256, 1), (335, 264, 256, 2), (335, 264, 256, 3), (335, 264, 256, 4),
                                     (335, 264, 256, 8), (2414, 1020, 512, 8), (9, 1020, 64, 4), (1, 8, 8, 1)])
def test_gemm_f32_scatter(M, N, K, n):
    """Every slot of every layout: each row lands bitwise at recv[row // R][slot][row % R] (the un-scattered EPI_F32 row, split-K
    off: the scatter switches the tail off), nothing else is written. M = 2414 at n = 8: R = 302, the last rank owns 300 rows;
    M = 9 at n = 4: R = 3, rank 3 owns none and its buffer stays untouched (the forward rejects such a layout, the GEMM does
    not). The CTA-pair kernel (M > 256) has its own EPI_F32 instantiation and must push the same bits."""
    g = torch.Generator().manual_seed(M + n)
    a = _rand_bf16(g, M, K, scale=0.5)
    w = _rand_bf16(g, N, K, scale=K ** -0.5)
    R = (M + n - 1) // n
    with _Options(splitk=0):
        ref = gemm_f32(a, w)
    for pair in (0, 1):
        for slot in range(n):
            recv = [sentinel_f32(n, R, N, device=DEV) for _ in range(n)]
            with _Options(pair=pair):
                gemm_scatter(a, w, recv, R, slot)
            err = scatter_mismatch(recv, scatter_expected(ref, n, R, slot))
            assert err is None, f"M={M} n={n} slot={slot} pair={pair}: {err}"
        if M == 9:
            assert is_sentinel(recv[3])


def test_gemm_f32_scatter_rejects_bad_layouts():
    L = _lib()
    g = torch.Generator().manual_seed(0)
    a = _rand_bf16(g, 10, 64)
    w = _rand_bf16(g, 16, 64)
    recv = [sentinel_f32(2, 4, 16, device=DEV) for _ in range(2)]
    for R, slot in ((4, 0), (0, 0), (5, 2), (5, -1)):  # 3 owners for 2 ranks, R = 0, slot past the buffers, negative slot
        with pytest.raises(L.MmdpError):
            gemm_scatter(a, w, recv, R, slot)
    torch.cuda.synchronize()
    assert all(is_sentinel(t) for t in recv), "a rejected call launches nothing"


# ---------------------------------------------------------------------------------------------------------------------------
# 2. residual add of a reduced partial sum
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,d,ldx,ldp", [(1, 8, 8, 8), (3, 1000, 1008, 1004), (5, 4096, 4096, 4100), (1, 4096, 4104, 4096)])
def test_resid_add_f32_bitwise(M, d, ldx, ldp):
    L = _lib()
    x, p = resid_inputs(M, d, seed=d + M)
    want = emulate_resid_add(x, p)
    xb = sentinel_bf16(M, ldx, device=DEV)
    xb[:, :d] = x.to(DEV)
    pb = sentinel_f32(M, ldp, device=DEV)
    pb[:, :d] = p.to(DEV)
    L.check(L.lib.mmdp_resid_add_f32(xb.data_ptr(), ldx, pb.data_ptr(), ldp, M, d, _stream()))
    got = xb[:, :d].cpu()
    bad = bitwise_mismatch(got, want)
    assert bad == 0, f"{bad} elements differ from bf16(x + bf16(partial))"
    assert is_sentinel(xb[:, d:]), "columns past d of x must stay untouched"
    for bad_d, bad_ldp in ((12, ldp), (d, 6)):
        with pytest.raises(L.MmdpError):
            L.check(L.lib.mmdp_resid_add_f32(xb.data_ptr(), ldx, pb.data_ptr(), bad_ldp, M, bad_d, _stream()))


# ---------------------------------------------------------------------------------------------------------------------------
# 3. reduce + residual + norm + broadcast, simulated ranks
# ---------------------------------------------------------------------------------------------------------------------------
GUARD = 2  # rows past the end of every xn / x_shard buffer that must keep their sentinel


class SimRanks:
    """The shared state of n tensor-parallel ranks on one device: every rank's activation buffer xn [M, d] bf16, flag array
    [2][8] and done counter, its rows of the residual stream x_shard [R, d], and (optionally) its receive buffers."""

    def __init__(self, n, M, d, n_recv=1):
        self.n, self.M, self.d = n, M, d
        self.R = (M + n - 1) // n
        self.xn = [sentinel_bf16(M + GUARD, d, device=DEV) for _ in range(n)]
        self.flags = [torch.zeros(2, 8, dtype=torch.int32, device=DEV) for _ in range(n)]
        self.done = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(n)]
        self.x = [sentinel_bf16(self.R + GUARD, d, device=DEV) for _ in range(n)]
        self.recv = [[sentinel_f32(n, self.R, d, device=DEV) for _ in range(n)] for _ in range(n_recv)]
        self._xn_arr, self._flag_arr = _ptrs(self.xn), _ptrs(self.flags)
        self._rows_bits = [None] * n

    def rows(self, r):
        return owned_rows(self.M, self.n, r)

    def reduce(self, my, n_src, w, eps, epoch, buf=0):
        """One mmdp_tp_reduce_norm call of rank `my`, under the safety rule: every flag of rank my's array (the waits of the
        call: phase 0 and 1 of every source) holds `epoch` before it, set on the same stream. The flags the call must write
        into the other ranks' arrays start at epoch - 1 and are checked afterwards, with the done counter."""
        L = _lib()
        r0, nr = self.rows(my)
        self.flags[my].fill_(epoch)
        for q in range(self.n):
            if q != my:
                self.flags[q][:, my] = epoch - 1
        L.check(L.lib.mmdp_tp_reduce_norm(self.recv[buf][my].data_ptr() if n_src else None, self.R, n_src, self._xn_arr,
                                          self._flag_arr, self.n, my, self.x[my].data_ptr(), w.data_ptr(), r0, nr, self.d, eps,
                                          epoch & 0xFFFFFFFF, self.done[my].data_ptr(), _stream()))
        for q in range(self.n):
            if q != my:
                f = self.flags[q][:, my].tolist()
                assert f == [epoch, epoch], f"rank {my}: flags it must set in rank {q}'s array are {f}, not the epoch {epoch}"
        assert int(self.done[my].item()) == 0, "the done counter must be back to 0 after the call"

    def check_broadcast(self, my):
        """Right after rank my's call, when the ranks run in order 0, 1, ... on buffers filled with the sentinel: rank my's rows
        are the same in every buffer, and every row after them (rows of ranks still to come, the guard rows) keeps the
        sentinel. The rows are kept for check_all_rows."""
        r0, nr = self.rows(my)
        mine = bits(self.xn[my][r0:r0 + nr]).clone()
        for q in range(self.n):
            assert torch.equal(bits(self.xn[q][r0:r0 + nr]), mine), f"rank {my}'s rows in rank {q}'s xn"
            assert is_sentinel(self.xn[q][r0 + nr:]), f"rank {my} wrote rows past its own into rank {q}'s xn"
        self._rows_bits[my] = mine

    def check_all_rows(self, what):
        """After every rank's call: every rank's rows in every buffer are still the ones its own call left (a later rank that
        also wrote rows below its own would change them), the guard rows keep the sentinel."""
        for q in range(self.n):
            for r in range(self.n):
                r0, nr = self.rows(r)
                assert torch.equal(bits(self.xn[q][r0:r0 + nr]), self._rows_bits[r]), \
                    f"{what}: rank {r}'s rows in rank {q}'s xn were overwritten after its call"
            assert is_sentinel(self.xn[q][self.M:]), f"{what}: guard rows of rank {q}'s xn"

    def assert_xn_identical(self, what):
        for r in range(1, self.n):
            assert torch.equal(bits(self.xn[r]), bits(self.xn[0])), f"{what}: rank {r}'s xn differs from rank 0's"


def _set_partials(sim, seed, buf=0):
    """Rank my's receive buffer, slot s = rank s's partial sums for rank my's rows (mixed sign and magnitude)."""
    for my in range(sim.n):
        _, nr = sim.rows(my)
        for s, p in enumerate(reduce_partials(sim.n, nr, sim.d, seed=seed * 131 + my)):
            sim.recv[buf][my][s, :nr] = p.to(DEV)


REDUCE_CASES = [  # (n, M, d): every NV template (d <= 2048 NV), partial thread groups (d / 8 not a multiple of 256), ragged last rank
    (1, 37, 256), (2, 75, 1000), (4, 130, 2048), (4, 61, 2056), (8, 2414, 4096), (2, 33, 5120), (8, 67, 8192), (1, 5, 8192),
]


@pytest.mark.parametrize("n,M,d", REDUCE_CASES)
def test_tp_reduce_norm(n, M, d):
    eps = 1e-5
    sim = SimRanks(n, M, d)
    g = torch.Generator().manual_seed(n * 1000 + d)
    w = (1 + 0.1 * torch.randn(d, generator=g)).to(torch.bfloat16).to(DEV)
    for my in range(n):
        _, nr = sim.rows(my)
        sim.x[my][:nr] = norm_inputs(nr, d, seed=my + d)[0].to(DEV) * 64
    order_pinned = 0
    for rnd, epoch in enumerate((5, 6)):  # the second call on the same buffers: the done counter was reset
        _set_partials(sim, seed=rnd + 10 * n)
        for t in sim.xn:
            t.copy_(sentinel_bf16(M + GUARD, d, device=DEV))
        for my in range(n):
            r0, nr = sim.rows(my)
            x0 = sim.x[my].clone()
            parts = [sim.recv[0][my][s, :nr] for s in range(n)]
            want = emulate_reduce(parts, x0[:nr])
            if n >= 3:  # the inputs make the rank order visible: the reversed order would disagree
                rev = emulate_reduce(parts, x0[:nr], order=list(reversed(range(n))))
                order_pinned += bitwise_mismatch(rev, want)
            sim.reduce(my, n, w, eps, epoch)
            got = sim.x[my]
            bad = bitwise_mismatch(got[:nr], want)
            assert bad == 0, f"rank {my}: x_shard differs from bf16(bf16(sum in rank order) + x) in {bad} elements"
            assert bitwise_mismatch(got[nr:], x0[nr:]) == 0, "rows past nrows of x_shard must stay untouched"
            assert_norm_exact(sim.xn[my][r0:r0 + nr], got[:nr], w, eps, f"n={n} d={d} rank {my} xn")
            sim.check_broadcast(my)
        sim.check_all_rows(f"n={n} d={d}")
    if n >= 3:
        assert order_pinned > 0


@pytest.mark.parametrize("n,M,d", [(1, 9, 1000), (4, 130, 4096), (8, 67, 8192)])
def test_tp_reduce_norm_without_partials(n, M, d):
    """n_src = 0 (the norm + broadcast after the embedding): x_shard is read, not written."""
    eps = 1e-5
    sim = SimRanks(n, M, d)
    w = norm_inputs(1, d, seed=d)[1].to(DEV)
    for my in range(n):
        _, nr = sim.rows(my)
        sim.x[my][:nr] = norm_inputs(nr, d, seed=3 * my + 1)[0].to(DEV)
    for my in range(n):
        r0, nr = sim.rows(my)
        x0 = sim.x[my].clone()
        sim.reduce(my, 0, w, eps, epoch=1)
        assert bitwise_mismatch(sim.x[my], x0) == 0, "n_src = 0 must leave x_shard untouched"
        assert_norm_exact(sim.xn[my][r0:r0 + nr], x0[:nr], w, eps, f"n_src=0 rank {my}")
        sim.check_broadcast(my)
    sim.check_all_rows("n_src=0")


def test_tp_reduce_norm_rejects_bad_arguments():
    """Host-side checks: nothing is launched, no flag or buffer is touched. The safety rule holds here too: every flag of every
    rank already holds the calls' epoch, and the host arrays have an entry for every rank index a bad call names (the extra
    entries point at rank 0's buffers), so even a call that launched could not wait on an unwritten flag."""
    L = _lib()
    n, M, d, epoch = 4, 40, 256, 1
    sim = SimRanks(n, M, d)
    w = torch.ones(d, dtype=torch.bfloat16, device=DEV)
    for f in sim.flags:
        f.fill_(epoch)
    x_before = [bits(t).clone() for t in sim.x]
    xn_arr = _ptrs(sim.xn + [sim.xn[0]] * (9 - n))
    flag_arr = _ptrs(sim.flags + [sim.flags[0]] * (9 - n))
    bad = [dict(n_src=1), dict(n_src=n, d=8200), dict(n_src=n, d=252), dict(n_src=n, nrows=0), dict(n_src=n, nrows=sim.R + 1),
           dict(n_src=n, my_rank=n), dict(n_src=0, n_ranks=9)]
    for kw in bad:
        n_src = kw.pop("n_src")
        r0, nr = sim.rows(0)
        args = dict(nrows=nr, d=d, my_rank=0, n_ranks=n)
        args.update(kw)
        with pytest.raises(L.MmdpError):
            L.check(L.lib.mmdp_tp_reduce_norm(sim.recv[0][0].data_ptr() if n_src else None, sim.R, n_src, xn_arr, flag_arr,
                                              args["n_ranks"], args["my_rank"], sim.x[0].data_ptr(), w.data_ptr(), r0, args["nrows"],
                                              args["d"], 1e-5, epoch, sim.done[0].data_ptr(), _stream()))
    torch.cuda.synchronize()
    assert all(bool((f == epoch).all()) for f in sim.flags), "the flags must still hold exactly the values set before the calls"
    assert all(int(c.item()) == 0 for c in sim.done)
    assert all(is_sentinel(t) for t in sim.xn), "a rejected call must not write xn"
    assert all(torch.equal(bits(t), b) for t, b in zip(sim.x, x_before)), "a rejected call must not write x_shard"


# ---------------------------------------------------------------------------------------------------------------------------
# 4. QKV + RoPE of a rank's heads
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h_local,B", [(2, 1), (2, 2), (4, 1), (4, 2), (16, 1), (16, 2)])
def test_qkv_rope_tp_shard(h_local, B):
    """Rank r of 2 owns heads [r h_local, (r + 1) h_local). Against the fp32 reference (the bounds of
    test_qkv_rope_and_attention), and - split-K off, the tiles cover the same rows of W in the same K order - bitwise equal to
    those heads' slice of mmdp_qkv_rope on the full weight."""
    from test_gpu_kernels import assert_ulp, ref_linear, ref_rope
    from mmada_parallel_b200.model import rope_tables
    L_ = _lib()
    tp, L = 2, 201  # Lpad = 208: the V^T pad columns exist and must stay zero
    H, da = tp * h_local, h_local * 128
    d, M, Lpad = H * 128, B * L, (L + 7) // 8 * 8
    g = torch.Generator().manual_seed(h_local * 10 + B)
    a = _rand_bf16(g, M, d)
    wq, wk, wv = (_rand_bf16(g, d, d, scale=d ** -0.5) for _ in range(3))
    cos, sin = (t.to(DEV) for t in rope_tables(128, 500000.0, L))
    with _Options(splitk=0):
        q_full, k_full, vt_full = _lib().qkv_rope(a, torch.cat([wq, wk, wv]), H, L, cos, sin)
        for r in range(tp):
            sl = slice(r * da, (r + 1) * da)
            wsh = torch.cat([wq[sl], wk[sl], wv[sl]]).contiguous()
            q = torch.empty(M, da, dtype=torch.bfloat16, device=DEV)
            k = torch.empty(M, da, dtype=torch.bfloat16, device=DEV)
            vt = torch.zeros(B, h_local, 128, Lpad, dtype=torch.bfloat16, device=DEV)
            L_.check(L_.lib.mmdp_qkv_rope_tp(a.data_ptr(), d, wsh.data_ptr(), M, d, h_local, L, Lpad, cos.data_ptr(), sin.data_ptr(),
                                             q.data_ptr(), k.data_ptr(), vt.data_ptr(), _stream()))
            qkv = ref_linear(a, wsh)
            pos = torch.arange(M, device=DEV) % L
            def pair_mag(x):
                xh = x.reshape(M, h_local, 2, 64).float().abs()
                return torch.maximum(xh[:, :, 0], xh[:, :, 1]).repeat(1, 1, 2).view(M, da)
            assert_ulp(q, ref_rope(qkv[:, :da].reshape(M, h_local, 128), cos[pos], sin[pos]).view(M, da), 2, "q rope", mag=pair_mag(qkv[:, :da]))
            assert_ulp(k, ref_rope(qkv[:, da:2 * da].reshape(M, h_local, 128), cos[pos], sin[pos]).view(M, da), 2, "k rope",
                       mag=pair_mag(qkv[:, da:2 * da]))
            assert_ulp(vt[..., :L].permute(0, 3, 1, 2).reshape(M, da), qkv[:, 2 * da:], 1, "v^T")
            assert bool((vt[..., L:] == 0).all())
            assert bitwise_mismatch(q, q_full[:, sl]) == 0, f"rank {r}: q differs from the full projection's heads"
            assert bitwise_mismatch(k, k_full[:, sl]) == 0, f"rank {r}: k differs from the full projection's heads"
            assert bitwise_mismatch(vt, vt_full[:, r * h_local:(r + 1) * h_local]) == 0, f"rank {r}: V^T differs"


# ---------------------------------------------------------------------------------------------------------------------------
# 5. mmdp_tp_forward at one rank, 6. TP = 2 / 4 / 8 op by op
# ---------------------------------------------------------------------------------------------------------------------------
ORACLE_ULPS_SIM = 5.0  # see test_tp_forward_simulated_ranks
TINY = dict(d_model=2048, n_heads=16, n_layers=2, mlp_hidden_size=4096, vocab_size=512, max_sequence_length=512)
_MODEL = {}


def _tiny_model():
    if not _MODEL:
        from oracle import llada
        cfg = llada.make_config(**TINY)
        _MODEL["cfg"] = cfg
        _MODEL["sd"] = llada.make_weights(cfg, seed=77)
    return _MODEL["cfg"], _MODEL["sd"]


def _shard(rank, tp):
    key = ("shard", rank, tp)
    if key not in _MODEL:
        from mmada_parallel_b200.tensor_parallel import shard_state_dict
        cfg, sd = _tiny_model()
        sh = shard_state_dict(sd, cfg.n_layers, cfg.n_heads, rank, tp, 0, cfg.vocab_size)
        _MODEL[key] = {k: v.to(DEV).contiguous() for k, v in sh.items()}
    return _MODEL[key]


def _ids(B, L):
    g = torch.Generator().manual_seed(B * 1000 + L)
    return torch.randint(0, TINY["vocab_size"], (B, L), generator=g)


def _oracle_hidden(B, L):
    key = ("oracle", B, L)
    if key not in _MODEL:
        from oracle import llada
        cfg, sd = _tiny_model()
        with torch.no_grad():
            _MODEL[key] = llada.forward_hidden(_ids(B, L), sd, cfg).reshape(B * L, -1)
    return _MODEL[key]


def _rope(L):
    from mmada_parallel_b200.model import rope_tables
    cos, sin = rope_tables(128, TINY.get("rope_theta", 500000.0), TINY["max_sequence_length"])
    return cos.to(DEV), sin.to(DEV)


def tp1_forward(B, L, n_chunks=1, chunk_rows0=0, epoch0=0):
    """mmdp_tp_forward with n_ranks = 1 on fresh buffers; returns (xn [M, d], epoch_out)."""
    L_ = _lib()
    cfg, _ = _tiny_model()
    w = _shard(0, 1)
    d, H, nl, ff = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size
    M, Lpad = B * L, (L + 7) // 8 * 8
    bf = dict(dtype=torch.bfloat16, device=DEV)
    keep = []
    layers = (L_.TpLayer * nl)()
    for i in range(nl):
        p = f"blocks.{i}."
        for name in ("wqkv", "wo", "w13", "w2", "attn_norm", "ff_norm"):
            setattr(layers[i], name, w[p + name].data_ptr())
    cos, sin = _rope(L)
    q, k, att = (torch.empty(M, d, **bf) for _ in range(3))
    h = torch.empty(M, ff, **bf)
    vt = torch.zeros(B, H, 128, Lpad, **bf)
    xn = sentinel_bf16(M, d, device=DEV)
    xn_arr = _ptrs([xn])
    c = L_.TpCtx()
    c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = d, H, ff, nl, 1, 0
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
    del keep
    return xn, int(out.value)


def ulp_errors(got, want):
    """Errors of `got` in bf16 ulp of the tensor's scale (max |want| x 2^-8): (max, mean, share of elements beyond 4 ulp).
    A non-finite element counts as an infinite error."""
    g, w = got.float().cpu(), want.float().cpu()
    ulp = w.abs().max().item() * 2.0 ** -8
    err = torch.where(torch.isfinite(g), (g - w).abs(), torch.full_like(g, math.inf)) / ulp
    return err.max().item(), err.mean().item(), (err > 4).float().mean().item()


@pytest.mark.parametrize("B,L", [(1, 301), (2, 150)])
def test_tp_forward_one_rank_vs_oracle(B, L):
    """ln_f(x) of every row, within 4 bf16 ulp of the tensor's scale of the CPU oracle (the bound of
    test_full_size_block_and_head_vs_oracle) with a mean error below half an ulp (on an H100: max 2.9 - 3.05, mean 0.30 - 0.33
    after two layers); repeated calls are bitwise equal; the epoch advances by 2 n_layers + 1, wrapping at 2^32."""
    cfg, _ = _tiny_model()
    xn, ep = tp1_forward(B, L, epoch0=7)
    assert ep == 7 + 2 * cfg.n_layers + 1
    mx, mean, _ = ulp_errors(xn, _oracle_hidden(B, L))
    print(f"[tp_forward 1 rank B={B} L={L}] vs oracle: max {mx:.2f} ulp, mean {mean:.4f} ulp")
    assert mx <= 4 and mean <= 0.5, (mx, mean)
    xn2, ep2 = tp1_forward(B, L, epoch0=2 ** 32 - 3)
    assert ep2 == (2 ** 32 - 3 + 2 * cfg.n_layers + 1) % 2 ** 32
    assert bitwise_mismatch(xn2, xn) == 0, "repeated forwards must be bitwise equal"


@pytest.mark.parametrize("chunk_rows0", [100, 150, 220])
def test_tp_forward_two_chunks_bitwise(chunk_rows0):
    """B = 2, L = 150: the chunk boundary inside batch row 0, exactly at the batch boundary, inside batch row 1. The second
    chunk's QKV epilogue runs with row0 = chunk_rows0 (positions and V^T addressed absolutely, q / k relative to the chunk).
    Split-K is off for both: which tiles a split-K tail takes depends on the launch's M, which differs between the schedules
    (the fp32 order of those tiles would differ); with it off every GEMM element has the same K order and the result must be
    bitwise that of one chunk."""
    with _Options(splitk=0):
        one, _ = tp1_forward(2, 150)
        two, ep = tp1_forward(2, 150, n_chunks=2, chunk_rows0=chunk_rows0, epoch0=100)
    cfg, _ = _tiny_model()
    assert ep == 100 + 2 * cfg.n_layers + 1
    diff = bits(two) != bits(one)
    assert not diff.any(), f"two chunks at {chunk_rows0}: {int(diff.sum())} elements differ (first row {int(diff.nonzero()[0, 0])})"


def sim_tp_forward(tp, B, L):
    """The per-layer sequence of mmdp_tp_forward (csrc/api.cu, mmdp_tp_forward: the embedding + n_src = 0 reduce at lines
    438-443, the column-parallel QKV + attention at 446-454, the attn_out scatter + ff_norm reduce at 461-462, the SwiGLU GEMM,
    ff_out scatter and the next norm's reduce at 463-465) issued from Python for every simulated rank in turn on one stream.
    A change to that sequence has to be mirrored here.
    After every reduce round all xn buffers must be bitwise identical. Returns rank 0's xn."""
    L_ = _lib()
    cfg, _ = _tiny_model()
    d, H, nl, ff, eps = cfg.d_model, cfg.n_heads, cfg.n_layers, cfg.mlp_hidden_size, cfg.rms_norm_eps
    Hl, ffl = H // tp, ff // tp
    da = Hl * 128
    M, Lpad = B * L, (L + 7) // 8 * 8
    sim = SimRanks(tp, M, d, n_recv=2)
    ws = [_shard(r, tp) for r in range(tp)]
    bf = dict(dtype=torch.bfloat16, device=DEV)
    q, k, att = (torch.empty(M, da, **bf) for _ in range(3))
    h = torch.empty(M, ffl, **bf)
    vt = torch.zeros(B, Hl, 128, Lpad, **bf)
    cos, sin = _rope(L)
    ids = _ids(B, L).to(DEV).view(-1)
    s = _stream()
    scale = 1.0 / math.sqrt(128.0)
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
            xn = sim.xn[r]
            L_.check(L_.lib.mmdp_qkv_rope_tp(xn.data_ptr(), d, ws[r][p + "wqkv"].data_ptr(), M, d, Hl, L, Lpad, cos.data_ptr(),
                                             sin.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), s))
            L_.check(L_.lib.mmdp_attention(q.data_ptr(), k.data_ptr(), vt.data_ptr(), att.data_ptr(), B, Hl, L, Lpad, scale, s))
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


@pytest.mark.parametrize("tp,B,L", [(2, 2, 150), (4, 2, 150), (4, 1, 301), (8, 1, 301), (8, 2, 150)])
def test_tp_forward_simulated_ranks(tp, B, L):
    """TP = 2 / 4 / 8 on one GPU, ragged row ownership (L = 301 at TP = 8: R = 38, the last rank owns 35). Every reduce round
    leaves all xn buffers bitwise identical (checked inside sim_tp_forward).

    The final xn against the one-rank mmdp_tp_forward: the only difference is the fp32 order of the row-parallel partial
    sums (K split over the ranks, summed in rank order). It is not a small difference after two layers: a bf16 rounding that
    flips in the first row-parallel GEMM feeds every later GEMM, the attention and the norms, and on an H100 (700 W) about
    73 % of the final elements differ, by 2.9 - 3.05 ulp of the tensor's scale at most and 0.27 - 0.28 ulp on average, at
    TP = 2, 4 and 8 alike - as far as either forward is from the CPU oracle (3.05 / 0.33). So the bound against the one-rank
    forward is that of the oracle comparison, 4 ulp with a mean below 0.35 ulp, not a tighter one. Against the oracle the
    same cascade put one element of TP = 4, B = 2, L = 150 at 4.34 ulp (the one-rank forward: 2.89), so the simulated ranks
    are held to ORACLE_ULPS_SIM = 5 ulp there, with at most 1 in 10^5 elements (6 of the 614 400) beyond 4 ulp - that one
    element was the only one beyond 4 ulp in the five cases - and the mean below 0.5 ulp (measured 0.30 - 0.33)."""
    got = sim_tp_forward(tp, B, L)
    one, _ = tp1_forward(B, L)
    mx1, mean1, _ = ulp_errors(got, one)
    mxo, meano, beyond = ulp_errors(got, _oracle_hidden(B, L))
    print(f"[simulated TP={tp} B={B} L={L}] vs one rank: max {mx1:.2f} ulp, mean {mean1:.4f} ulp, "
          f"differing {(bits(got) != bits(one)).float().mean().item():.4f} | vs oracle: max {mxo:.2f} ulp, mean {meano:.4f} ulp, "
          f"beyond 4 ulp {beyond * got.numel():.0f} elements")
    assert mx1 <= 4 and mean1 <= 0.35, f"from the one-rank forward: max {mx1:.2f}, mean {mean1:.3f} ulp"
    assert mxo <= ORACLE_ULPS_SIM and meano <= 0.5, f"from the oracle: max {mxo:.2f}, mean {meano:.3f} ulp"
    assert beyond <= 1e-5, f"from the oracle: {beyond * got.numel():.0f} elements beyond 4 ulp"


# ---------------------------------------------------------------------------------------------------------------------------
# 7. every dispatch branch of mmdp_rmsnorm
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("warp", [1, 0])
@pytest.mark.parametrize("d", [256, 512, 1024, 2048, 4096, 3072, 8192, 12288])
def test_rmsnorm_every_branch_exact(d, warp):
    """d = 256 ... 4096: one warp per row (rmsnorm_warp_kernel<1..16>); other d and rmsnorm_warp = 0: one CTA per row, the row
    held in registers up to d = 8192 and re-read at d = 12288. Strided x and y (ldx, ldy > d), the `rows` gather and an M that is
    not a multiple of 8; boundary-aware exact (tp_ops_ref.norm_expected)."""
    L_ = _lib()
    eps = 1e-5
    M, ldx, ldy = 37, d + 24, d + 8
    x, w = norm_inputs(M, d, seed=d + warp)
    xs = sentinel_bf16(M, ldx, device=DEV)   # rows of stride ldx; the pad columns are never read
    xs[:, :d] = x.to(DEV)
    w = w.to(DEV)
    rows = torch.tensor([5, 0, M - 1, 17, 5, 30, 2], dtype=torch.int32, device=DEV)
    try:
        L_.check(L_.lib.mmdp_set_option(b"rmsnorm_warp", warp))
        for sel in (None, rows):
            n = M if sel is None else sel.numel()
            y = sentinel_bf16(n, ldy, device=DEV)
            L_.check(L_.lib.mmdp_rmsnorm(xs.data_ptr(), ldx, None if sel is None else sel.data_ptr(), w.data_ptr(), y.data_ptr(), ldy,
                                         n, d, eps, _stream()))
            src = xs[:, :d] if sel is None else xs[sel.long(), :d]
            assert_norm_exact(y[:, :d], src, w, eps, f"rmsnorm d={d} warp={warp} rows={sel is not None}")
            assert is_sentinel(y[:, d:]), "columns past d of y must stay untouched"
    finally:
        L_.check(L_.lib.mmdp_set_option(b"rmsnorm_warp", 1))
