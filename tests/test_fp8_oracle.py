"""The FP8 oracle (oracle/fp8.py) that defines the opt-in e4m3 precision of the block linears: quantiser properties, the
GEMM formula against an fp64 evaluation, and the FP8 forward of the tiny model against the bf16 forward (a sanity check
of the scheme, not a parity claim)."""
import math

import torch
import torch.nn.functional as F

from helpers import load_golden, tiny_cfg_and_weights
from oracle import fp8, llada


def e4m3_ulp(y: torch.Tensor) -> torch.Tensor:
    """Spacing of e4m3 values at |y| (3 mantissa bits, normal from 2^-6, subnormal spacing 2^-9)."""
    e = torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -6)))
    return torch.exp2(e - 3)


def test_group_max_maps_to_448_and_zero_group():
    torch.manual_seed(0)
    x = (torch.randn(5, 512) * 3).to(torch.bfloat16)
    x[1, 128:256] = 0
    x[2, 300] = -1000.0
    q, s = fp8.quantize_fp8(x, 128)
    assert q.dtype == torch.float8_e4m3fn and tuple(q.shape) == (5, 512) and tuple(s.shape) == (4, 5)
    qf = q.float().view(5, 4, 128)
    xf = x.float().view(5, 4, 128)
    idx = xf.abs().argmax(-1, keepdim=True)
    top = qf.gather(-1, idx).squeeze(-1)
    zero = xf.abs().amax(-1) == 0
    assert torch.equal(top[~zero].abs(), torch.full_like(top[~zero], 448.0))
    assert torch.equal(torch.sign(top[~zero]), torch.sign(xf.gather(-1, idx).squeeze(-1)[~zero]))
    assert bool(zero[1, 1]) and float(s[1, 1]) == 1.0 and bool((qf[1, 1] == 0).all())
    assert float(qf[2, 2].min()) == -448.0


def test_rounding_error_is_half_an_e4m3_ulp():
    torch.manual_seed(1)
    x = (torch.randn(64, 1024) * torch.logspace(-3, 2, 1024)).to(torch.bfloat16)
    for group in (128, 1024):
        q, s = fp8.quantize_fp8(x, group)
        sx = s.t().repeat_interleave(group, dim=1).double()              # [rows, K]
        y = (x.float() / sx.float()).double()                              # the fp32 quotient that was rounded
        err = (q.double() - y).abs()
        assert bool((err <= 0.5 * e4m3_ulp(y)).all()), group
        # in units of x: |q*s - x| <= half an ulp of x/s, times s (plus the rounding of the fp32 quotient)
        assert bool(((q.double() * sx - x.double()).abs() <= 0.5 * e4m3_ulp(y) * sx * (1 + 2.0 ** -20) + 2.0 ** -149).all())


def test_groups_are_independent():
    torch.manual_seed(2)
    x = torch.randn(3, 512).to(torch.bfloat16)
    q0, s0 = fp8.quantize_fp8(x, 128)
    x2 = x.clone()
    x2[:, 256:384] *= 1000
    q1, s1 = fp8.quantize_fp8(x2, 128)
    keep = torch.ones(512, dtype=torch.bool)
    keep[256:384] = False
    assert torch.equal(q0.view(torch.uint8)[:, keep], q1.view(torch.uint8)[:, keep])
    assert torch.equal(s0[[0, 1, 3]], s1[[0, 1, 3]]) and not torch.equal(s0[2], s1[2])


def test_no_nan_on_extreme_inputs():
    big = torch.finfo(torch.bfloat16).max
    tiny = torch.finfo(torch.bfloat16).smallest_normal
    x = torch.zeros(4, 256, dtype=torch.bfloat16)
    x[0, :128] = big
    x[0, 5] = -big
    x[0, 128:] = torch.tensor([tiny * 2.0 ** -k for k in range(1, 8)] * 19)[:128].to(torch.bfloat16)  # subnormals only
    x[1, :] = -0.0
    x[1, 7] = 0.0
    x[2, :] = torch.linspace(-1, 1, 256).to(torch.bfloat16)
    x[2, 3] = tiny * 2.0 ** -7                                           # subnormal next to normal values
    x[3, :128] = big
    x[3, 128] = tiny * 2.0 ** -3
    for group in (128, 256):
        q, s = fp8.quantize_fp8(x, group)
        assert torch.isfinite(q.float()).all() and torch.isfinite(s).all() and bool((s > 0).all())
        assert float(q.float().abs().max()) == 448.0
    q, s = fp8.quantize_fp8(x, 128)
    assert bool((q[0, 128:].float().abs() > 0).any()), "a subnormal-only group still quantises to non-zero values"
    assert bool((q[1].float() == 0).all()) and float(s[0, 1]) == 1.0


def _fp64_formula(qa, sa, qw, sw):
    M, K = qa.shape
    N = qw.shape[0]
    a = qa.double().view(M, K // 128, 128)
    w = qw.double().view(N, K // 128, 128)
    exact = torch.einsum("mgk,ngk,gm->mn", a, w, sa.double()) * sw.double()[None, :]
    abssum = torch.einsum("mgk,ngk,gm->mn", a.abs(), w.abs(), sa.double()) * sw.double().abs()[None, :]
    return exact, abssum


def test_linear_fp8_vs_fp64():
    torch.manual_seed(3)
    for M, N, K in [(1, 8, 128), (37, 72, 512), (130, 256, 1536)]:
        x = (torch.randn(M, K) * 2).to(torch.bfloat16)
        wt = (torch.randn(N, K) * 0.05).to(torch.bfloat16)
        qa, sa = fp8.quantize_fp8(x, 128)
        qw, sw = fp8.quantize_fp8(wt, K)
        got = fp8.linear_fp8(qa, sa, qw, sw[0])
        assert got.dtype == torch.float32 and tuple(got.shape) == (M, N)
        exact, abssum = _fp64_formula(qa, sa, qw, sw[0])
        # fp32 recursive-summation bound: 127 additions in a group, one scale product, K/128 group additions, one weight scale
        u = 2.0 ** -24
        bound = (128 + K // 128 + 2) * u * abssum
        assert bool(((got.double() - exact).abs() <= bound + 1e-30).all()), (M, N, K)


def test_tiny_forward_fp8_vs_bf16_oracle():
    g = load_golden("forward_tiny.pt")
    cfg, sd = tiny_cfg_and_weights(g["meta"])
    ids = g["ids"]
    with torch.no_grad():
        ref = llada.forward_logits(ids, sd, cfg).float()
        got = fp8.forward_logits_fp8(ids, sd, cfg).float()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    rel_rms = ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    rel_max = ((got - ref).abs().max() / ref.abs().max()).item()
    agree = (got.argmax(-1) == ref.argmax(-1)).float().mean().item()
    print(f"[fp8 oracle] tiny model logits vs bf16 oracle: relative RMS {rel_rms:.4f}, max/scale {rel_max:.4f}, argmax agreement {agree:.3f}")
    # e4m3 keeps 3 mantissa bits: one linear with both operands quantised is ~4 % off in relative RMS, and this random-weight
    # model carries that through 2 blocks and 8 linears to ~10 % (measured); a scheme error (wrong scale, lost group) is far larger
    assert rel_rms < 0.25 and rel_max < 0.5
    assert math.isfinite(rel_rms)


def test_cached_oracle_linear_hook():
    """llada.CachedOracleModel's `linear` hook: its default is the reference's bf16 F.linear (the same bits as the hook spelled out,
    and as the real reference on the token-cache golden's calls), and with fp8.linear_hook the full forward is
    fp8.forward_logits_fp8 bit for bit, as is a partial forward that recomputes every position."""
    g = load_golden("forward_tiny.pt")
    cfg, sd = tiny_cfg_and_weights(g["meta"])
    t = load_golden("token_cache_tiny.pt")
    default = llada.CachedOracleModel(cfg, sd)
    spelled = llada.CachedOracleModel(cfg, sd, linear=lambda x, name: F.linear(x, sd[name]))
    for case in t["cases"]:
        for st in case["steps"]:
            a = default(st["ids"], to_compute_mask=st["mask"], cat=case["cat"]).logits
            b = spelled(st["ids"], to_compute_mask=st["mask"], cat=case["cat"]).logits
            assert torch.equal(a, b) and torch.equal(a[:, :, st["cols"]], st["logits_cols"]), case["name"]
    wq = fp8.quantize_weights(sd)
    om = llada.CachedOracleModel(cfg, sd, linear=fp8.linear_hook(wq))
    ids = g["ids"]
    with torch.no_grad():
        want = fp8.forward_logits_fp8(ids, sd, cfg, wq)
    assert torch.equal(om(ids, cat="x").logits, want)
    assert torch.equal(om(ids, to_compute_mask=torch.ones_like(ids, dtype=torch.bool), cat="x").logits, want)
