"""The opt-in FP8 (e4m3) precision of the block linears on the H100 against its definition, oracle/fp8.py: the quantiser bit for
bit, the e4m3 GEMM within the bf16-ulp bounds of test_gpu_kernels.py (1 plain, 2 residual, 3 SwiGLU) plus the accumulation
error of the e4m3 tensor-core sum, the tiny model's forward and generation loops, one block at production shapes, and the
isolation of a bf16 context from an FP8 one."""
import contextlib
import io
from types import SimpleNamespace

import pytest
import torch

from helpers import GpuBackedOracleModel, load_golden, tiny_cfg_and_weights, tiny_gpu_model
from oracle import fp8
from oracle import generate as G
from test_gpu_kernels import bf

pytestmark = pytest.mark.gpu


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def u8(q):
    return q.view(torch.uint8)


def assert_ulp(got, want, ulps, what, mag=None, abssum=None):
    """The bound of test_gpu_kernels.assert_ulp - |got - want| <= ulps bf16 spacings at the magnitude of the rounded quantities -
    plus the accumulation error of the e4m3 tensor-core sum: inside a k-block it keeps about 13 bits of its absolute-value sum
    (`abssum`: linear_fp8 of |qa|, |qw|), not fp32's 24, so a few roundings per million move one ulp further than in the bf16
    GEMM (measured: 146 of 9.9 M at K = 12288). The share of differing roundings is reported and bounded loosely."""
    g, w = got.float(), want.float()
    assert not torch.isnan(g).any(), what
    scale = w.abs().max().clamp_min(1e-20)
    ref_mag = w.abs() if mag is None else torch.maximum(w.abs(), mag.float().abs())
    tol = ulps * torch.maximum(ref_mag, scale / 64) * 2.0 ** -7
    if abssum is not None:
        tol = tol + abssum.float() * 2.0 ** -12
    bad = (g - w).abs() > tol
    differ = (g != w).float().mean().item()
    print(f"[{what}] max err {float((g - w).abs().max()):.3g}, roundings differing from the oracle: {differ:.4f}")
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} outside {ulps} ulp; max abs err {float((g - w).abs().max())}"
    assert g.numel() < 1024 or differ < 0.25, f"{what}: too many roundings differ ({differ})"


def _abssum(qa, sa, qw, sw):
    """linear_fp8 on the absolute values: the magnitude the tensor-core accumulation error scales with."""
    return _want(qa.float().abs().to(torch.float8_e4m3fn), sa, qw.float().abs().to(torch.float8_e4m3fn), sw.abs())


# ---------------------------------------------------------------------------------------------------------------------
# 1. quantiser: bytes and scales bit-identical to the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _hard_input(rows, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, K, generator=g) * torch.logspace(-2, 1, K)
    x[3, 17] = 30000.0                                    # one huge value in a row
    x[5, :] = 0.0                                         # an all-zero row (all groups zero)
    x[6, 128:256] = 0.0                                   # one all-zero group
    x[6, 130] = -0.0
    tiny = torch.finfo(torch.bfloat16).smallest_normal
    x[7, :128] = tiny * 2.0 ** -torch.arange(1, 129).remainder(7).add(1).float()   # a subnormal-only group
    x[8, ::5] = tiny * 2.0 ** -3                          # subnormals among normal values
    x[9, 0] = torch.finfo(torch.bfloat16).max
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("rows,K", [(333, 512), (1, 256), (130, 4096)])
def test_quantize_bit_exact(rows, K):
    from mmada_parallel_b200 import _lib
    rows_in = max(rows, 10)
    x = _hard_input(rows_in, K, rows + K)[:rows].contiguous()
    for group in (128, K):
        q, s = _lib.quantize_fp8(x.cuda(), group)
        qo, so = fp8.quantize_fp8(x, group)
        assert torch.equal(u8(q).cpu(), u8(qo)), (rows, K, group, "bytes")
        assert torch.equal(s.cpu(), so), (rows, K, group, "scales")


def test_quantize_strided_and_wide():
    from mmada_parallel_b200 import _lib
    big = _hard_input(200, 1024 + 192, 7)
    x = big[:, 64:64 + 1024]                              # row stride 1216 > K
    xg = big.cuda()[:, 64:64 + 1024]
    assert xg.stride(0) == 1216
    q, s = _lib.quantize_fp8(xg, 128)
    qo, so = fp8.quantize_fp8(x.contiguous(), 128)
    assert torch.equal(u8(q).cpu(), u8(qo)) and torch.equal(s.cpu(), so)
    x = big[:, 4:4 + 1024]                                # 8-byte aligned rows: the warp-per-group kernel
    q, s = _lib.quantize_fp8(big.cuda()[:, 4:4 + 1024], 128)
    qo, so = fp8.quantize_fp8(x.contiguous(), 128)
    assert torch.equal(u8(q).cpu(), u8(qo)) and torch.equal(s.cpu(), so)
    w = _hard_input(64, 12288, 8)                         # a weight row of ff_out: group = K = 12288
    q, s = _lib.quantize_fp8(w.cuda(), 12288)
    qo, so = fp8.quantize_fp8(w, 12288)
    assert torch.equal(u8(q).cpu(), u8(qo)) and torch.equal(s.cpu(), so)
    with pytest.raises(_lib.MmdpError):
        _lib.quantize_fp8(torch.zeros(4, 200, dtype=torch.bfloat16, device="cuda"), 100)   # group not a multiple of 128


# ---------------------------------------------------------------------------------------------------------------------
# 2. e4m3 GEMM against linear_fp8 on the same quantised operands
# ---------------------------------------------------------------------------------------------------------------------
def _operands(M, N, K, seed, wstd=0.05):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = bf(torch.randn(M, K, device="cuda", generator=g) * 0.5)
    w = bf(torch.randn(N, K, device="cuda", generator=g) * wstd)
    from mmada_parallel_b200 import _lib
    qa, sa = _lib.quantize_fp8(a, 128)
    qw, sw = _lib.quantize_fp8(w, K)
    return qa, sa, qw, sw[0].contiguous()


def _want(qa, sa, qw, sw):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fp8.linear_fp8(qa, sa, qw, sw)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("M,N,K", [(1, 8, 128), (333, 264, 256), (2414, 4096, 4096), (2414, 4096, 12288)])
def test_gemm_fp8_plain_and_resid(M, N, K):
    """(2414, 4096, 12288) is the accumulator-precision check: ff_out's K. Without the per-k-block promotion into fp32 the
    e4m3 tensor-core accumulator would drift past 1 bf16 ulp."""
    from mmada_parallel_b200 import _lib
    qa, sa, qw, sw = _operands(M, N, K, M + N + K)
    lin = _want(qa, sa, qw, sw)
    acc_err = _abssum(qa, sa, qw, sw)
    got = _lib.gemm_fp8(qa, sa, qw, sw)
    assert_ulp(got, bf(lin), 1, f"gemm_fp8 {M}x{N}x{K}", abssum=acc_err)
    assert torch.equal(got, _lib.gemm_fp8(qa, sa, qw, sw)), "bitwise repeatable"
    r = bf(torch.randn(M, N, device="cuda"))
    want = bf(bf(lin).float() + r.float())
    assert_ulp(_lib.gemm_fp8(qa, sa, qw, sw, _lib.EPI_RESID, resid=r), want, 2, f"gemm_fp8 resid {M}x{N}x{K}", mag=bf(lin), abssum=acc_err)
    r2 = r.clone()
    _lib.gemm_fp8(qa, sa, qw, sw, _lib.EPI_RESID, resid=r2, out=r2)
    assert_ulp(r2, want, 2, "resid in place", mag=bf(lin), abssum=acc_err)
    # the FP8 kernel has no split-K tail: the split-K option leaves it unchanged
    try:
        _lib.lib.mmdp_set_gemm_splitk(3)
        assert torch.equal(got, _lib.gemm_fp8(qa, sa, qw, sw))
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)


def _interleave64(t1, t3):
    ff = t1.shape[0]
    out = torch.empty((2 * ff,) + tuple(t1.shape[1:]), dtype=t1.dtype, device=t1.device)
    out.view(ff // 64, 2, 64, *t1.shape[1:])[:, 0] = t1.view(ff // 64, 64, *t1.shape[1:])
    out.view(ff // 64, 2, 64, *t1.shape[1:])[:, 1] = t3.view(ff // 64, 64, *t1.shape[1:])
    return out


@pytest.mark.parametrize("M,ff,K", [(300, 512, 512), (2414, 12288, 4096)])
def test_gemm_fp8_swiglu(M, ff, K):
    from mmada_parallel_b200 import _lib
    qa, sa, q1, s1 = _operands(M, ff, K, 11 + M, wstd=0.08)
    _, _, q3, s3 = _operands(M, ff, K, 12 + M, wstd=0.08)
    got = _lib.gemm_fp8(qa, sa, u8(_interleave64(u8(q1), u8(q3))).view(torch.float8_e4m3fn), _interleave64(s1, s3), _lib.EPI_SWIGLU)
    assert got.shape == (M, ff)
    g1, g3 = bf(_want(qa, sa, q1, s1)), bf(_want(qa, sa, q3, s3))
    want = bf(bf(torch.nn.functional.silu(g1.float())).float() * g3.float())
    acc_err = torch.maximum(_abssum(qa, sa, q1, s1), _abssum(qa, sa, q3, s3))
    assert_ulp(got, want, 3, f"gemm_fp8 swiglu {M}x{2 * ff}x{K}", abssum=acc_err)


def _on_gpu_fp32(fn):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _assert_as_close_as_torch(err, err_e, ulp, what):
    """4 bf16 ulp of the tensor's scale, the bound of the bf16 forward tests, or - where the quantisation makes that unreachable
    for any implementation - no further from the CPU oracle than the same oracle code run by torch on the GPU (x1.5): an e4m3
    rounding that flips on a one-ulp difference of its bf16 input moves the output by up to an e4m3 step, and torch on the GPU
    flips such roundings just as the native path does (measured: 16 ulp max at production shapes)."""
    assert torch.isfinite(err).all(), what
    assert err.max().item() <= max(4 * ulp, 1.5 * err_e.max().item()), (what, "max", err.max().item() / ulp, err_e.max().item() / ulp)
    assert err.mean().item() <= 1.5 * err_e.mean().item() + 0.02 * ulp, (what, "mean", err.mean().item() / ulp, err_e.mean().item() / ulp)


# ---------------------------------------------------------------------------------------------------------------------
# 3. tiny model in FP8 against oracle.fp8
# ---------------------------------------------------------------------------------------------------------------------
_FP8_CACHE = {}


def tiny_fp8_model(meta, cls=None, max_batch=3):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    cls = cls or LLaDAForMultiModalGeneration
    key = (cls.__name__, meta["weight_seed"], tuple(sorted(meta["tiny"].items())), max_batch)
    if key not in _FP8_CACHE:
        cfg, sd = tiny_cfg_and_weights(meta)
        if cls.__name__ == "MMadaModelLM":
            cfg.mask_token_id = 126336
        m = cls(cfg, max_seq_len=cfg.max_sequence_length, max_batch=max_batch, precision="fp8")
        m.load_state_dict(sd)
        _FP8_CACHE[key] = (m, cfg, sd)
    return _FP8_CACHE[key]


def test_precision_argument():
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    g = load_golden("forward_tiny.pt")
    m, _, _ = tiny_fp8_model(g["meta"])
    assert m.precision == "fp8"
    assert tiny_gpu_model(g["meta"])[0].precision == "bf16"
    cfg, _ = tiny_cfg_and_weights(g["meta"])
    with pytest.raises(ValueError):
        LLaDAForMultiModalGeneration(cfg, max_seq_len=128, max_batch=1, precision="fp16")


def test_tiny_forward_vs_fp8_oracle():
    g = load_golden("forward_tiny.pt")
    model, cfg, sd = tiny_fp8_model(g["meta"])
    lg = model(g["ids"], infer=True, use_cache=False).logits
    assert lg.dtype == torch.bfloat16 and tuple(lg.shape) == (1, g["ids"].shape[1], cfg.vocab_size)
    with torch.no_grad():
        want = fp8.forward_logits_fp8(g["ids"], sd, cfg).float()[0]
        eager = _on_gpu_fp32(lambda: fp8.forward_logits_fp8(g["ids"].cuda(), {k: v.cuda() for k, v in sd.items()}, cfg)).float()[0].cpu()
    got = lg[0].float().cpu()
    ulp = want.abs().max().item() * 2.0 ** -8
    err, err_e = (got - want).abs(), (eager - want).abs()
    print(f"[fp8 tiny] logits vs oracle.fp8 on the CPU: max {err.max().item() / ulp:.2f} ulp of the scale, mean {err.mean().item() / ulp:.4f} "
          f"| the oracle by torch on the GPU: max {err_e.max().item() / ulp:.2f}, mean {err_e.mean().item() / ulp:.4f}")
    _assert_as_close_as_torch(err, err_e, ulp, "tiny logits")
    # CFG batch rows are independent
    lg2 = model(g["ids2"], infer=True, use_cache=False).logits
    assert torch.equal(lg2[0], lg[0])


def test_tiny_restricted_head_window_and_cache():
    from mmada_parallel_b200 import _lib
    g = load_golden("forward_tiny.pt")
    model, cfg, _ = tiny_fp8_model(g["meta"])
    ids = g["ids2"].cuda()
    L = ids.shape[1]
    full = model(ids, infer=True).logits.view(2 * L, -1)
    rows_a = torch.tensor([3, 10, L + 5, 2 * L - 1], dtype=torch.int32, device="cuda")
    rows_b = torch.arange(5, 37, dtype=torch.int32, device="cuda")
    a, b = model.forward_rows(ids, rows_a=rows_a, rows_b=rows_b, col0_b=126356, ncols_b=8192)
    assert torch.equal(a, full[rows_a.long()])
    assert torch.equal(b, full[rows_b.long()][:, 126356:126356 + 8192])
    # row window of the last block: bit-identical with attention's KV-split tail off (as for bf16)
    one = ids[0:1].contiguous()
    ra = torch.arange(40, 60, dtype=torch.int32, device="cuda")
    rb = torch.arange(20, 40, dtype=torch.int32, device="cuda")
    try:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 0))
        fa, fb = model.forward_rows(one, rows_a=ra, rows_b=rb, col0_b=126356, ncols_b=8192)
        wa, wb = model.forward_rows(one, rows_a=ra, rows_b=rb, col0_b=126356, ncols_b=8192, row_window=(20, 60))
    finally:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))
    assert torch.equal(fa, wa) and torch.equal(fb, wb)
    model.raise_device_errors()
    # token cache: the full forward that fills the caches gives the dense forward's logits
    model.caching(True)
    try:
        cached = model(one, infer=True, use_cache=True, cat="x").logits
        dense = model(one, infer=True, use_cache=False).logits
        assert torch.equal(cached, dense)
    finally:
        model.caching(False)


# ---------------------------------------------------------------------------------------------------------------------
# 4. production shapes: one block at d=4096 / ff=12288 / 32 heads / L=2414 plus the restricted heads
# ---------------------------------------------------------------------------------------------------------------------
def test_full_size_block_and_head_vs_fp8_oracle():
    """FP8 on the H100 against oracle.fp8 on the CPU with the same weights (mirrors test_full_size_block_and_head_vs_oracle):
    max and mean error no larger than 1.5x those of the same oracle code run by torch on the GPU (max: or 4 bf16 ulp of the
    tensor's scale), see _assert_as_close_as_torch."""
    import time
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from oracle import llada
    from test_gpu_model import _device_view_bf16
    cfg = llada.make_config(d_model=4096, n_heads=32, n_layers=1, mlp_hidden_size=12288, vocab_size=134656, max_sequence_length=2432)
    g = torch.Generator(device="cuda").manual_seed(2025)
    d, ff, V, L = 4096, 12288, 134656, 2414

    def rnd(*s, std):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16)

    p = "model.transformer.blocks.0."
    sd = {"model.transformer.wte.weight": rnd(V, d, std=0.02), "model.transformer.ff_out.weight": rnd(V, d, std=d ** -0.5),
          "model.transformer.ln_f.weight": (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)}
    for n, shape, std in [("q_proj", (d, d), d ** -0.5), ("k_proj", (d, d), d ** -0.5), ("v_proj", (d, d), d ** -0.5),
                          ("attn_out", (d, d), d ** -0.5), ("ff_proj", (ff, d), d ** -0.5), ("up_proj", (ff, d), d ** -0.5),
                          ("ff_out", (d, ff), ff ** -0.5)]:
        sd[p + n + ".weight"] = rnd(*shape, std=std)
    sd[p + "attn_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)
    sd[p + "ff_norm.weight"] = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).to(torch.bfloat16)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=2432, max_batch=1, precision="fp8")
    m.load_state_dict(sd)
    ids = torch.randint(0, 126000, (1, L), device="cuda", generator=g)
    text_rows = torch.arange(2157, 2413, dtype=torch.int32, device="cuda")
    img_rows = torch.arange(1100, 1100 + 1024, dtype=torch.int32, device="cuda")
    a, b = m.forward_rows(ids, rows_a=text_rows, rows_b=img_rows, col0_b=126356, ncols_b=8192)
    hidden = _device_view_bf16(_lib.lib.mmdp_model_hidden(m._h), L * d).view(L, d).clone()
    torch.cuda.synchronize()

    def oracle(w, ids_):
        with torch.no_grad():
            wq = fp8.quantize_weights(w)
            x = torch.nn.functional.embedding(ids_, w["model.transformer.wte.weight"])
            pos_sin, pos_cos = llada.rotary_tables(128, cfg.rope_theta, L)
            x = fp8.block_forward_fp8(x, w, wq, p, cfg, pos_sin.to(x.device), pos_cos.to(x.device))
            xn = llada.rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)[0]
            head = w["model.transformer.ff_out.weight"]
            return x[0], torch.nn.functional.linear(xn[2157:2413], head), torch.nn.functional.linear(xn[1100:1100 + 1024], head[126356:126356 + 8192])

    t0 = time.time()
    x_o, a_o, b_o = oracle({k: v.cpu() for k, v in sd.items()}, ids.cpu())
    print(f"[full-size fp8 oracle] CPU block + heads: {time.time() - t0:.1f} s")
    x_e, a_e, b_e = _on_gpu_fp32(lambda: oracle(sd, ids))

    failures = []

    def check(got, eager, want, what):
        gq, eq, wq = got.float().cpu(), eager.float().cpu(), want.float()
        scale = wq.abs().max().item()
        ulp = scale * 2.0 ** -8
        err, err_e = (gq - wq).abs(), (eq - wq).abs()
        print(f"[full-size fp8] {what}: scale {scale:.3f} | native vs CPU oracle: max {err.max().item() / ulp:.2f} ulp, mean "
              f"{err.mean().item() / ulp:.4f} ulp | torch-on-GPU vs CPU oracle: max {err_e.max().item() / ulp:.2f} ulp, "
              f"mean {err_e.mean().item() / ulp:.4f} ulp")
        try:
            _assert_as_close_as_torch(err, err_e, ulp, what)
        except AssertionError as e:
            failures.append(e.args)

    check(hidden, x_e, x_o, "residual stream after the block")
    check(a, a_e, a_o, "text-row logits")
    check(b, b_e, b_o, "image-row codebook logits")
    assert not failures, failures


# ---------------------------------------------------------------------------------------------------------------------
# 5. generation in FP8
# ---------------------------------------------------------------------------------------------------------------------
def _args(lay):
    return {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}


def test_generate_ti2ti_fp8_lockstep_with_oracle():
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    t = load_golden("trajectory_a_tiny.pt")
    model, _, _ = tiny_fp8_model(t["meta"])
    lay = t["layout"]
    backed = GpuBackedOracleModel(model)
    for run in t["runs"][:2]:
        torch.manual_seed(run["global_seed"])
        img_o, txt_o = G.generate_ti2ti(backed, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                        stable_sort=True, **_args(lay), **run["kwargs"])
        outs = []
        for _ in range(2):
            torch.manual_seed(run["global_seed"])
            with quiet():
                outs.append(generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                           **_args(lay), **run["kwargs"]))
        assert outs[0] == outs[1], (run["name"], "two runs with the same generator")
        assert outs[0] == (img_o, txt_o), run["name"]


def test_interleave_generate_fp8():
    from mmada_parallel_b200.mmada import MMadaModelLM
    t = load_golden("trajectory_m_tiny.pt")
    model, _, _ = tiny_fp8_model(t["meta"], cls=MMadaModelLM, max_batch=2)
    assert model.precision == "fp8"
    conf = SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=t["num_vq_tokens"], codebook_size=8192)),
                           dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=t["max_seq_length"])))

    class Tok:
        bos_token_id = t["bos"]

        def __len__(self):
            return t["text_vocab_len"]

    up = SimpleNamespace(text_tokenizer=Tok())
    run = t["runs"][0]
    outs = [model.interleave_generate(input_ids=t["input_ids"], uncond_input_ids=t["uncond_input_ids"],
                                      reserved_token_mapping={"<|soi|>": t["soi"], "<|eoi|>": t["eoi"]},
                                      generator=torch.Generator().manual_seed(run["seed"]), config=conf, uni_prompting=up,
                                      **run["kwargs"]) for _ in range(2)]
    img_o, txt_o = G.interleave_generate(GpuBackedOracleModel(model), t["input_ids"], t["uncond_input_ids"], soi_id=t["soi"],
                                         eoi_id=t["eoi"], bos_id=t["bos"], mask_id=t["mask_id"], num_vq_tokens=t["num_vq_tokens"],
                                         codebook_size=8192, max_seq_length=t["max_seq_length"], text_vocab_len=t["text_vocab_len"],
                                         generator=torch.Generator().manual_seed(run["seed"]), **run["kwargs"])
    (img0, txt0), (img1, txt1) = outs
    assert torch.equal(img0, img1) and torch.equal(txt0, txt1), "two runs with the same generator"
    assert torch.equal(txt0.cpu(), txt_o) and torch.equal(img0.cpu(), img_o)


# ---------------------------------------------------------------------------------------------------------------------
# 6. isolation: an FP8 context leaves a bf16 context's results untouched
# ---------------------------------------------------------------------------------------------------------------------
def test_bf16_context_unchanged_by_fp8_context():
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    g = load_golden("forward_tiny.pt")
    ref_model, cfg, sd = tiny_gpu_model(g["meta"])
    before = ref_model(g["ids2"], infer=True).logits.clone()
    m8 = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=2, precision="fp8")
    m8.load_state_dict(sd)
    lg8 = m8(g["ids2"], infer=True).logits
    m8.forward_rows(g["ids2"].cuda(), rows_a=torch.arange(0, 16, dtype=torch.int32, device="cuda"))
    after = ref_model(g["ids2"], infer=True).logits
    assert torch.equal(before, after)
    assert not torch.equal(lg8, after), "the FP8 context computes its own (quantised) logits"
    del m8
    assert torch.equal(before, ref_model(g["ids2"], infer=True).logits)
