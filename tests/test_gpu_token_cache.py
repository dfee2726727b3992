"""The token-cache forward (mmdp_model_forward_cached: `model.caching(True)`, then `model(ids, infer=True, use_cache=True,
to_compute_mask=mask, cat=key)`) op by op at production shapes, through the test hooks of include/mmdp_testing_cache.h:

  - the QKV + RoPE GEMM with a position map, bf16 and e4m3: compact row r is token pos[r] of batch row r / Tq; q stays compact,
    k rows and V^T columns are scattered into the caches at that position. Against the fp32 reference of test_qkv_rope_and_attention
    (oracle.fp8.linear_fp8 for e4m3) at the mapped positions, with every unselected cache row / column checked bit for bit
    against its sentinel, the V^T pad columns against zero, and bit for bit against the dense launch (Tq = L, no map) at the same
    positions: without the split-K tail a GEMM row does not depend on M, and rotary only on the position;
  - attention of Tq query rows against all L cached keys, against an fp64 softmax(QK^T)V, on shapes that reach every branch of
    the KV-split planner (plan_split_tail, restated below), and bit for bit against the dense launch with the split tail off;
  - negative controls: plausible bugs of this mode computed in torch land outside the bounds the kernels are held to;
  - one production-size layer through the model against oracle.llada.CachedOracleModel on the CPU, in bf16 and in FP8.
"""
import ctypes as C
import math
import os
import re
import time

import pytest
import torch

from test_gpu_kernels import assert_attention_close, assert_ulp, attn_version, bf, ref_linear, ref_rope  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

_vp, _i, _f = C.c_void_p, C.c_int, C.c_float
# name -> argtypes (every hook returns int); must list every symbol declared in include/mmdp_testing_cache.h
HOOKS = {
    "mmdp_testing_qkv_rope_cached": [_i, _vp, _i, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp],
    "mmdp_testing_attention_cached": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp],
}

H, D, L0 = 32, 4096, 2414
SCALE = 1.0 / math.sqrt(128.0)


def declared_cache_symbols():
    from helpers import ROOT
    src = open(os.path.join(ROOT, "include", "mmdp_testing_cache.h")).read()
    return sorted(set(re.findall(r"MMDP_API[^;(]*?\b(mmdp_[a-z0-9_]+)\s*\(", src)))


def hooks():
    """libmmdp.so with the argument types of the token-cache hooks set."""
    from mmada_parallel_b200 import _lib
    for name, args in HOOKS.items():
        fn = getattr(_lib.lib, name)
        fn.restype, fn.argtypes = _i, args
    return _lib.lib


def call(name, *args):
    from mmada_parallel_b200 import _lib
    _lib.check(getattr(hooks(), name)(*args, _lib.stream_ptr()))


def p(t):
    return None if t is None else t.data_ptr()


class Options:
    """Sets library options for a block and restores their defaults (split-K mode 2, attention split tail on, generation 6)."""
    DEFAULTS = {"gemm_splitk": 2, "attn_split_tail": 1, "attn_version": 6}

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        from mmada_parallel_b200 import _lib
        for k, v in self.kw.items():
            _lib.check(_lib.lib.mmdp_set_option(k.encode(), v))

    def __exit__(self, *exc):
        from mmada_parallel_b200 import _lib
        for k in self.kw:
            _lib.check(_lib.lib.mmdp_set_option(k.encode(), self.DEFAULTS[k]))


# ---------------------------------------------------------------------------------------------------------------------
# position maps
# ---------------------------------------------------------------------------------------------------------------------
def random_positions(g, L, n, exclude=()):
    pool = torch.tensor(sorted(set(range(L)) - set(exclude)))
    return sorted(pool[torch.randperm(len(pool), generator=g)[:n]].tolist())


def store_path_map():
    """Compact rows laid out so that the staged V^T store meets each of its forms (8-row groups at compact rows 8i):
    a 16-byte store needs 8 consecutive positions of one batch row from a multiple of 8, everything else takes element stores."""
    rows = [0, 3, 9, 17, 20, 33, 40, 41]          # rows 0-7: scattered, position 0
    rows += list(range(64, 72))                   # rows 8-15: an aligned run of 8 -> vector store
    rows += list(range(128, 144))                 # rows 16-31: an aligned run of 16 -> two vector stores
    rows += list(range(203, 211))                 # rows 32-39: a run of 8 from 203 % 8 = 3 -> element stores
    rows += [300, 301, 302]                       # rows 40-42
    rows += list(range(400, 408))                 # rows 43-50: aligned positions straddling two row groups
    rows += [500, 600, 700, 800, 900]             # rows 51-55
    rows += list(range(1000, 1008))               # rows 56-63: aligned run -> vector store
    rows += list(range(1013, 1021))               # rows 64-71: a run of 8 from 1013 % 8 = 5
    rows += list(range(2400, 2408))               # rows 72-79: aligned run -> vector store
    rows += [L0 - 1]                              # row 80: the last position
    return [rows]


def straddle_map(g):
    """B = 2, Tq = 300 (Tq % 8 = 4): the 8-row group at compact rows 296-303 holds positions 1200-1203 of batch row 0 and
    1204-1207 of batch row 1 - consecutive and aligned, so only the batch-row check keeps it off the 16-byte V^T store."""
    b0 = random_positions(g, 1200, 296) + [1200, 1201, 1202, 1203]
    b1 = [1204, 1205, 1206, 1207] + [1208 + x for x in random_positions(g, L0 - 1208, 296)]
    return [b0, b1]


def qkv_cases():
    g = torch.Generator().manual_seed(7)
    return {
        "tq1": (L0, [random_positions(g, L0, 1)]),
        "tq7": (L0, [random_positions(g, L0, 7)]),
        "tq300": (L0, [random_positions(g, L0, 300)]),
        "tq2414_arange": (L0, [list(range(L0))]),
        "store_paths": (L0, store_path_map()),
        "b2_straddle": (L0, straddle_map(g)),
        "l333": (333, [[0] + random_positions(g, 320, 40, exclude=(0,)) + list(range(320, 328)) + [332]]),
        "l333_arange": (333, [list(range(333))]),
    }


QKV_CASES = qkv_cases()


# ---------------------------------------------------------------------------------------------------------------------
# QKV + RoPE with a position map
# ---------------------------------------------------------------------------------------------------------------------
def pair_mag(x):
    """Rotary mixes element i with i +- 64 of the same head: both magnitudes bound the rounding error."""
    M = x.shape[0]
    xh = x.view(M, -1, 2, 64).float().abs()
    return torch.maximum(xh[:, :, 0], xh[:, :, 1]).repeat(1, 1, 2).view(M, -1)


class QkvCase:
    """Operands of one position-mapped QKV launch: the dense activations of all B*L tokens, the compact rows the map selects,
    the caches filled with random sentinels (V^T pad columns zero)."""

    def __init__(self, name):
        from mmada_parallel_b200.model import rope_tables
        L, maps = QKV_CASES[name]
        self.name, self.L, self.B, self.Tq = name, L, len(maps), len(maps[0])
        self.Lpad = (L + 7) // 8 * 8
        g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
        self.pos = torch.tensor(sum(maps, []), dtype=torch.int32, device="cuda")
        self.b = torch.arange(self.B, device="cuda").repeat_interleave(self.Tq)
        self.rows = self.b * L + self.pos.long()                                 # cache row of each compact row
        self.a_dense = bf(torch.randn(self.B * L, D, device="cuda", generator=g))
        self.a = self.a_dense[self.rows].contiguous()
        self.w = bf(torch.randn(3 * D, D, device="cuda", generator=g) / math.sqrt(D))
        self.cos, self.sin = (t.cuda() for t in rope_tables(128, 500000.0, L))
        self.k0 = bf(torch.randn(self.B * L, D, device="cuda", generator=g))
        self.vt0 = torch.zeros(self.B, H, 128, self.Lpad, dtype=torch.bfloat16, device="cuda")
        self.vt0[..., :L] = bf(torch.randn(self.B, H, 128, L, device="cuda", generator=g))

    def run(self, a, sa=None, w=None, sw=None, dense=False):
        """One launch into fresh copies of the sentinel caches -> (q, kcache, vtcache)."""
        Tq, pos = (self.L, None) if dense else (self.Tq, self.pos)
        q = torch.full((self.B * Tq, D), float("nan"), dtype=torch.bfloat16, device="cuda")
        k, vt = self.k0.clone(), self.vt0.clone()
        w = self.w if w is None else w
        precision = 1 if a.dtype == torch.float8_e4m3fn else 0
        call("mmdp_testing_qkv_rope_cached", precision, p(a), a.stride(0), p(sa), p(w), p(sw), self.B, Tq, p(pos), D, H, self.L,
             self.Lpad, p(self.cos), p(self.sin), p(q), p(k), p(vt))
        return q, k, vt

    def v_at(self, vt):
        """V^T columns of the mapped positions as rows [B*Tq, D]."""
        return vt[self.b, :, :, self.pos.long()].reshape(-1, D)

    def reference(self, qkv):
        """q, k at the mapped positions and v, from the bf16 projections [B*Tq, 3D]."""
        pos = self.pos.long()
        M = qkv.shape[0]
        q = ref_rope(qkv[:, :D].view(M, H, 128), self.cos[pos], self.sin[pos]).view(M, D)
        k = ref_rope(qkv[:, D:2 * D].view(M, H, 128), self.cos[pos], self.sin[pos]).view(M, D)
        return q, k, qkv[:, 2 * D:]

    def assert_untouched(self, k, vt):
        """Cache rows / V^T columns the map does not select keep their sentinels bit for bit; pad columns stay zero."""
        keep = torch.ones(self.B * self.L, dtype=torch.bool, device="cuda")
        keep[self.rows] = False
        assert torch.equal(k[keep].view(torch.int16), self.k0[keep].view(torch.int16)), f"{self.name}: a k cache row outside the map was written"
        keep_v = keep.view(self.B, self.L)
        got_v, want_v = vt[..., :self.L].permute(0, 3, 1, 2), self.vt0[..., :self.L].permute(0, 3, 1, 2)
        assert torch.equal(got_v[keep_v].view(torch.int16), want_v[keep_v].view(torch.int16)), f"{self.name}: a V^T column outside the map was written"
        assert bool((vt[..., self.L:] == 0).all()), f"{self.name}: V^T pad columns must stay zero"

    def assert_matches_dense(self, got, dense):
        """q, k, V^T at position p equal the dense launch's at p, bit for bit."""
        (q, k, vt), (qd, kd, vtd) = got, dense
        assert torch.equal(q, qd[self.rows]), f"{self.name}: q differs from the dense launch"
        assert torch.equal(k[self.rows], kd[self.rows]), f"{self.name}: k differs from the dense launch"
        assert torch.equal(self.v_at(vt), self.v_at(vtd)), f"{self.name}: V^T differs from the dense launch"


def _err_ulp(got, want, mag=None):
    """Max and mean |got - want| in bf16 ulps of max(|want|, |mag|, scale / 64) - the unit of assert_ulp's bound (for the log)."""
    w = want.float()
    ref_mag = w.abs() if mag is None else torch.maximum(w.abs(), mag.float().abs())
    e = (got.float() - w).abs() / (torch.maximum(ref_mag, w.abs().max() / 64) * 2.0 ** -7)
    return f"max {e.max().item():.2f} ulp, mean {e.mean().item():.4f} ulp"


@pytest.mark.parametrize("name", list(QKV_CASES))
def test_qkv_cached_bf16(name):
    """(a) against the fp32 reference (2 ulp with the rotary pair magnitude for q / k, 1 ulp for V^T), nothing else written,
    split-K mode 0 and 3 identical (the position map switches the tail off); (b) bit for bit with the dense launch."""
    c = QkvCase(name)
    with Options(gemm_splitk=0):
        got = c.run(c.a)
        dense = c.run(c.a_dense, dense=True)
    with Options(gemm_splitk=3):
        got3 = c.run(c.a)
    for x, y in zip(got, got3):
        assert torch.equal(x, y), f"{name}: split-K mode 3 changed a position-mapped launch"
    q, k, vt = got
    qkv = ref_linear(c.a, c.w)
    q_ref, k_ref, v_ref = c.reference(qkv)
    print(f"[qkv bf16 {name}] q {_err_ulp(q, q_ref, pair_mag(qkv[:, :D]))} | k {_err_ulp(k[c.rows], k_ref, pair_mag(qkv[:, D:2 * D]))} "
          f"| v {_err_ulp(c.v_at(vt), v_ref)}")
    assert_ulp(q, q_ref, 2, f"{name} q rope", mag=pair_mag(qkv[:, :D]))
    assert_ulp(k[c.rows], k_ref, 2, f"{name} k rope", mag=pair_mag(qkv[:, D:2 * D]))
    assert_ulp(c.v_at(vt), v_ref, 1, f"{name} v^T")
    c.assert_untouched(k, vt)
    c.assert_matches_dense(got, dense)


@pytest.mark.parametrize("name", list(QKV_CASES))
def test_qkv_cached_fp8(name):
    """(c) the e4m3 launch against oracle.fp8.linear_fp8 + rotary with the abssum bound of test_gpu_fp8.assert_ulp, nothing else
    written; (b) bit for bit with the dense e4m3 launch (activation scales are per row, so quantising the compact rows gives
    the dense rows' bytes)."""
    from mmada_parallel_b200 import _lib
    from test_gpu_fp8 import _abssum, _want
    from test_gpu_fp8 import assert_ulp as assert_ulp_fp8
    c = QkvCase(name)
    qa, sa = _lib.quantize_fp8(c.a, 128)
    qd, sd = _lib.quantize_fp8(c.a_dense, 128)
    qw, sw = _lib.quantize_fp8(c.w, D)
    sw = sw[0].contiguous()
    got = c.run(qa, sa, qw, sw)
    dense = c.run(qd, sd, qw, sw, dense=True)
    q, k, vt = got
    lin = _want(qa, sa, qw, sw)
    acc = _abssum(qa, sa, qw, sw)
    qkv = bf(lin)
    q_ref, k_ref, v_ref = c.reference(qkv)
    # rotary output t1 cos - t2 sin: the accumulation errors of both inputs reach it, |cos| + |sin| <= sqrt 2
    acc_q, acc_k = (math.sqrt(2) * pair_mag(acc[:, r * D:(r + 1) * D]) for r in (0, 1))
    print(f"[qkv fp8 {name}] q {_err_ulp(q, q_ref, pair_mag(qkv[:, :D]))} | k {_err_ulp(k[c.rows], k_ref, pair_mag(qkv[:, D:2 * D]))} "
          f"| v {_err_ulp(c.v_at(vt), v_ref)}")
    assert_ulp_fp8(q, q_ref, 2, f"{name} fp8 q rope", mag=pair_mag(qkv[:, :D]), abssum=acc_q)
    assert_ulp_fp8(k[c.rows], k_ref, 2, f"{name} fp8 k rope", mag=pair_mag(qkv[:, D:2 * D]), abssum=acc_k)
    assert_ulp_fp8(c.v_at(vt), v_ref, 1, f"{name} fp8 v^T", abssum=acc[:, 2 * D:])
    c.assert_untouched(k, vt)
    c.assert_matches_dense(got, dense)


# ---------------------------------------------------------------------------------------------------------------------
# attention of Tq query rows against L cached keys
# ---------------------------------------------------------------------------------------------------------------------
ATTN_CASES = [(1, 300), (1, 640), (1, 100), (2, 2100), (2, 1)]  # (B, Tq) at H = 32, L = 2414


def plan_split_tail(tiles, n_kvb, slots):
    """csrc/attention.cu plan_split_tail with the split tail on and one KV length -> (branch, split tiles, pieces per tile)."""
    def fit(want):
        sp = min(8, want, n_kvb // 2)
        while sp >= 2 and (sp - 1) * -(-n_kvb // sp) >= n_kvb:
            sp -= 1
        return sp
    if tiles > slots and tiles % slots and (tiles % slots) * 4 <= slots:
        sp = fit(slots // (tiles % slots))
        if sp >= 2:
            return "partial-wave split", tiles % slots, sp
    elif tiles * 2 <= slots:
        sp = fit(slots // tiles)
        if sp >= 2:
            return "every tile split", tiles, sp
    return "no split", 0, 1


def attn_plan(B, Tq, kbkv):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return plan_split_tail(-(-Tq // 128) * H * B, -(-L0 // kbkv), sms)


def test_attention_cases_reach_every_split_branch():
    """The attention cases reach each branch of plan_split_tail with Lq != L on this device, for both kernel generations
    (128- and 64-key blocks); the B = 2 partial wave lies wholly in batch row 1 (the b * Lq addressing of the combine pass)."""
    for kbkv in (128, 64):
        plans = {case: attn_plan(*case, kbkv) for case in ATTN_CASES}
        print(f"[plan_split_tail, {kbkv}-key blocks] " + "; ".join(f"B={B} Tq={Tq}: {pl[0]} ({pl[1]} tiles x {pl[2]})"
                                                             for (B, Tq), pl in plans.items()))
        assert {pl[0] for pl in plans.values()} == {"no split", "partial-wave split", "every tile split"}, plans
        assert any(B == 2 and pl[0] == "partial-wave split" for (B, _), pl in plans.items()), plans
        for (B, Tq), (branch, n_split, _) in plans.items():
            if B == 2 and branch == "partial-wave split":
                n_qt = -(-Tq // 128)
                assert n_qt * H * B - n_split >= n_qt * H, "the split tiles should all be in batch row 1"


def attn_operands(B, Tq, seed):
    """Dense q / k / v of all B*L tokens, V^T with zero pad columns, and the compact rows of a random sorted map per batch row."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Lpad = (L0 + 7) // 8 * 8
    q_dense = bf(torch.randn(B * L0, D, device="cuda", generator=g))
    k = bf(torch.randn(B * L0, D, device="cuda", generator=g))
    v = bf(torch.randn(B * L0, D, device="cuda", generator=g))
    vt = torch.zeros(B, H, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    vt[..., :L0] = v.view(B, L0, H, 128).permute(0, 2, 3, 1)
    gc = torch.Generator().manual_seed(seed)
    pos = torch.cat([torch.randperm(L0, generator=gc)[:Tq].sort().values for _ in range(B)]).cuda()
    rows = torch.arange(B, device="cuda").repeat_interleave(Tq) * L0 + pos
    return q_dense, k, v, vt, rows


def attention_cached(q, k, vt, B, Tq):
    out = torch.full_like(q, float("nan"))
    call("mmdp_testing_attention_cached", p(q), p(k), p(vt), p(out), B, H, L0, vt.shape[-1], Tq, SCALE)
    return out


def attention_ref(q, k, v, B, Tq, Lk=L0):
    """fp64 softmax(q k^T * scale) v per batch row: q [B*Tq, D] against k / v [B*Lk, D] -> [B*Tq, D]."""
    out = []
    for b in range(B):
        qh = q[b * Tq:(b + 1) * Tq].double().view(Tq, H, 128).transpose(0, 1)
        kh = k[b * Lk:(b + 1) * Lk].double().view(Lk, H, 128).transpose(0, 1)
        vh = v[b * Lk:(b + 1) * Lk].double().view(Lk, H, 128).transpose(0, 1)
        out.append((torch.softmax(qh @ kh.transpose(-1, -2) * SCALE, dim=-1) @ vh).transpose(0, 1).reshape(Tq, D))
    return torch.cat(out).float()


def _attn_err(o, o_ref):
    rms = o_ref.pow(2).mean(-1, keepdim=True).sqrt()
    e = (o.float() - o_ref).abs() / (torch.maximum(o_ref.abs(), rms) * 2.0 ** -8)
    return f"max {e.max().item():.2f} ulp, mean {e.mean().item():.4f} ulp"


@pytest.mark.parametrize("B,Tq", ATTN_CASES)
def test_attention_cached(B, Tq, attn_version):
    """(d) Tq < L query rows against all L keys: the fp64 reference within assert_attention_close's bound with the split tail on
    and off; off, each row equals the same position's row of the dense launch bit for bit (same row arithmetic, same KV order);
    on vs off within the same relative bound. (The absolute split-vs-unsplit bound of test_attention_full_length_relative_error,
    2^-8 of the output's max, does not hold here: that launch, 608 tiles on 132 SMs, has no split tile, while splitting every
    tile moves single elements by 2 bf16 ulp of their own magnitude.)"""
    q_dense, k, v, vt, rows = attn_operands(B, Tq, 1000 * B + Tq)
    q = q_dense[rows].contiguous()
    o_ref = attention_ref(q, k, v, B, Tq)
    with Options(attn_split_tail=0):
        o0 = attention_cached(q, k, vt, B, Tq)
        od = attention_cached(q_dense, k, vt, B, L0)
    with Options(attn_split_tail=1):
        o1 = attention_cached(q, k, vt, B, Tq)
    branch = attn_plan(B, Tq, 128 if attn_version == 6 else 64)
    print(f"[attention v{attn_version} B={B} Tq={Tq}, {branch[0]}] vs fp64, split tail off: {_attn_err(o0, o_ref)} | on: "
          f"{_attn_err(o1, o_ref)} | on vs off: {_attn_err(o1, o0.float())}")
    assert torch.equal(o0, od[rows]), "a row of the compact launch differs from the dense launch's row at its position"
    assert_attention_close(o0, o_ref, f"cached attention B{B} Tq{Tq}, split tail off")
    assert_attention_close(o1, o_ref, f"cached attention B{B} Tq{Tq}, split tail on")
    # A split piece rounds its probabilities to bf16 relative to its own running max, so split rows differ from unsplit ones by
    # P roundings that average out over the row (measured: up to 3.2 ulp of max(|o|, row rms), mean 0.29 ulp, every tile split).
    assert_attention_close(o1, o0.float(), f"cached attention B{B} Tq{Tq}, split tail on vs off")


# ---------------------------------------------------------------------------------------------------------------------
# negative controls
# ---------------------------------------------------------------------------------------------------------------------
def test_bounds_reject_plausible_bugs():
    """(e) Each plausible bug of the token-cache launches, computed in torch on the B = 2 production case, lands outside the
    bound its kernel is held to above: rotary at the compact row instead of the mapped position, attention over only the Tq
    selected keys, batch row 1 attending to batch row 0's keys, a V^T column written one position off."""
    c = QkvCase("b2_straddle")
    qkv = ref_linear(c.a, c.w)
    q_ref, _, v_ref = c.reference(qkv)
    compact = torch.arange(c.Tq, device="cuda").repeat(c.B)
    q_bug = ref_rope(qkv[:, :D].view(-1, H, 128), c.cos[compact], c.sin[compact]).view(-1, D)
    with pytest.raises(AssertionError):
        assert_ulp(q_bug, q_ref, 2, "rotary at the compact row", mag=pair_mag(qkv[:, :D]))
    vt_bug = c.vt0.clone()
    vt_bug[c.b, :, :, (c.pos.long() + 1).clamp_max(c.L - 1)] = v_ref.view(-1, H, 128)
    with pytest.raises(AssertionError):
        assert_ulp(c.v_at(vt_bug), v_ref, 1, "V^T one position off")

    B, Tq = 2, 300
    q_dense, k, v, _, rows = attn_operands(B, Tq, 77)
    q = q_dense[rows]
    o_ref = attention_ref(q, k, v, B, Tq)
    with pytest.raises(AssertionError):
        assert_attention_close(attention_ref(q, k[rows], v[rows], B, Tq, Lk=Tq), o_ref, "attention over the selected keys only")
    k0, v0 = k[:L0].repeat(2, 1), v[:L0].repeat(2, 1)
    with pytest.raises(AssertionError):
        assert_attention_close(attention_ref(q, k0, v0, B, Tq), o_ref, "batch row 1 reads batch row 0's keys")


# ---------------------------------------------------------------------------------------------------------------------
# one production-size layer through the model against the token-cache oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_one_layer_token_cache_vs_oracle(precision):
    """(f) d = 4096, ff = 12288, 32 heads, L = 2414, one layer, a 16384-row vocabulary (the filling forward computes logits
    for all L rows): caching(True), one full forward, then partial forwards of 300 random positions and of 640 positions with
    a run of 200 consecutive ones, new token ids at the recomputed positions. Against oracle.llada.CachedOracleModel on the CPU
    (FP8: its linear hook oracle.fp8.linear_hook) with the yardstick of test_full_size_block_and_head_vs_oracle: 4 bf16 ulp of
    the scale and a mean error no worse than 1.5x that of the same oracle run by torch on the GPU (FP8: test_gpu_fp8's
    _assert_as_close_as_torch)."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from oracle import fp8, llada
    from test_gpu_fp8 import _assert_as_close_as_torch, _on_gpu_fp32
    d, ff, V, L = D, 12288, 16384, L0
    cfg = llada.make_config(d_model=d, n_heads=H, n_layers=1, mlp_hidden_size=ff, vocab_size=V, max_sequence_length=2432)
    g = torch.Generator(device="cuda").manual_seed(2026)

    def rnd(*s, std):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16)

    pre = "model.transformer.blocks.0."
    sd = {"model.transformer.wte.weight": rnd(V, d, std=0.02), "model.transformer.ff_out.weight": rnd(V, d, std=d ** -0.5),
          "model.transformer.ln_f.weight": (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)}
    for n, shape, std in [("q_proj", (d, d), d ** -0.5), ("k_proj", (d, d), d ** -0.5), ("v_proj", (d, d), d ** -0.5),
                          ("attn_out", (d, d), d ** -0.5), ("ff_proj", (ff, d), d ** -0.5), ("up_proj", (ff, d), d ** -0.5),
                          ("ff_out", (d, ff), ff ** -0.5)]:
        sd[pre + n + ".weight"] = rnd(*shape, std=std)
    sd[pre + "attn_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)
    sd[pre + "ff_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)

    gc = torch.Generator().manual_seed(5)
    m300 = torch.zeros(1, L, dtype=torch.bool)
    m300[0, torch.randperm(L, generator=gc)[:300]] = True
    m640 = torch.zeros(1, L, dtype=torch.bool)
    m640[0, 1000:1200] = True
    m640[0, torch.tensor(random_positions(gc, L, 440, exclude=range(1000, 1200)))] = True
    ids = torch.randint(0, V, (1, L), generator=gc)
    steps = [(ids, None)]
    for mask in (m300, m640):
        ids = torch.where(mask, torch.randint(0, V, (1, L), generator=gc), ids)
        steps.append((ids, mask))

    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=2432, max_batch=1, precision=precision)
    m.load_state_dict(sd)
    m.caching(True)
    try:
        got = [m(i.cuda(), infer=True, use_cache=True, to_compute_mask=None if k is None else k.cuda(), cat="t").logits.clone()
               for i, k in steps]
    finally:
        m.caching(False)
    m.raise_device_errors()

    def run_oracle(w, dev):
        hook = fp8.linear_hook(fp8.quantize_weights(w)) if precision == "fp8" else None
        om = llada.CachedOracleModel(cfg, w, linear=hook)
        with torch.no_grad():
            return [om(i.to(dev), to_compute_mask=None if k is None else k.to(dev), cat="t").logits.clone() for i, k in steps]

    t0 = time.time()
    want = run_oracle({k: v.cpu() for k, v in sd.items()}, "cpu")
    print(f"[token-cache layer {precision}] CPU oracle, one full and two partial forwards: {time.time() - t0:.1f} s")
    eager = _on_gpu_fp32(lambda: run_oracle(sd, "cuda"))

    failures = []
    for s, (what, (_, mask)) in enumerate(zip(("full forward", "partial, 300 positions", "partial, 640 positions"), steps)):
        sel = torch.ones(1, L, dtype=torch.bool) if mask is None else mask
        gq, eq, wq = got[s].cpu()[sel].float(), eager[s].cpu()[sel].float(), want[s][sel].float()
        ulp = wq.abs().max().item() * 2.0 ** -8
        err, err_e = (gq - wq).abs(), (eq - wq).abs()
        print(f"[token-cache layer {precision}] {what}: native vs CPU oracle max {err.max().item() / ulp:.2f} ulp, mean "
              f"{err.mean().item() / ulp:.4f} ulp | torch on the GPU vs CPU oracle max {err_e.max().item() / ulp:.2f} ulp, mean "
              f"{err_e.mean().item() / ulp:.4f} ulp")
        if mask is not None:
            assert torch.equal(got[s][~mask.cuda()], got[s - 1][~mask.cuda()]), "positions not recomputed keep their cached logits"
        try:
            if precision == "fp8":
                _assert_as_close_as_torch(err, err_e, ulp, what)
            else:
                assert torch.isfinite(gq).all(), what
                assert err.max().item() <= 4 * ulp, (what, "max", err.max().item() / ulp)
                assert err.mean().item() <= 1.5 * err_e.mean().item() + 0.02 * ulp, (what, "mean", err.mean().item() / ulp)
        except AssertionError as e:
            failures.append(e.args)
    assert not failures, failures
