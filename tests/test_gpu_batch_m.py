"""Packed forwards with per-sequence last-block row windows, and the variant-M batch loop, on the H100: the windowed packed
attention kernel against `attention_packed` and an fp32 reference, `forward_rows_packed(row_windows=)` against unwindowed and
per-sequence forwards (bf16, FP8, grouped-query + bias, production shapes), and `interleave_generate_batch` against sequential
`interleave_generate` calls."""
import contextlib
import math
from types import SimpleNamespace

import pytest
import torch

from helpers import load_golden, tiny_cfg_and_weights
from test_gpu_kernels import assert_attention_close

pytestmark = pytest.mark.gpu

SCALE = 1.0 / math.sqrt(128.0)


@pytest.fixture(params=[6, 7])
def attn_version(request):
    """Both attention kernel generations (6: 128-key blocks, the default; 7: 64-key blocks)."""
    from mmada_parallel_b200 import _lib
    _lib.check(_lib.lib.mmdp_set_option(b"attn_version", request.param))
    yield request.param
    _lib.check(_lib.lib.mmdp_set_option(b"attn_version", 6))


@contextlib.contextmanager
def split_tail(on):
    from mmada_parallel_b200 import _lib
    _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", int(on)))
    try:
        yield
    finally:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))


@contextlib.contextmanager
def splits_off():
    """GEMM split-K tail and attention KV-split tail off: which tiles they touch depends on the problem size, so only without
    them is a row bit-identical whatever else the launch computes."""
    from mmada_parallel_b200 import _lib
    _lib.lib.mmdp_set_gemm_splitk(0)
    _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 0))
    try:
        yield
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))


# ---------------------------------------------------------------------------------------------------------------------
# 1. windowed packed attention
# ---------------------------------------------------------------------------------------------------------------------
# windows at row offsets 0, 1, 127, 128 and 129, one-row windows, whole sequences and M's text window (the last 256 of 2341)
_LENS = [1, 129, 300, 1000, 2414, 700, 2341, 130]
_WINDOWS = [(0, 1), (1, 129), (127, 128), (128, 1000), (129, 2414), (0, 700), (2085, 2341), (129, 130)]


@pytest.mark.parametrize("H,Hkv", [(4, 4), (32, 8)])
def test_packed_window_attention(H, Hkv, attn_version):
    from mmada_parallel_b200 import _lib
    lens, wins = _LENS, _WINDOWS
    d, dkv, M, n = H * 128, Hkv * 128, sum(lens), len(lens)
    Lpad = (max(lens) + 7) // 8 * 8
    torch.manual_seed(11 + H)
    q = torch.randn(M, d, device="cuda").to(torch.bfloat16)
    k = torch.randn(M, dkv, device="cuda").to(torch.bfloat16)
    v = torch.randn(M, dkv, device="cuda").to(torch.bfloat16)
    vt = torch.zeros(n, Hkv, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    offs = [sum(lens[:i]) for i in range(n)]
    for i, (o, L) in enumerate(zip(offs, lens)):
        vt[i, :, :, :L] = v[o:o + L].view(L, Hkv, 128).permute(1, 2, 0)
    full, win = {}, {}
    for split in (0, 1):
        with split_tail(split):
            full[split] = (_lib.attention_packed(q, k, vt, lens, H, SCALE) if H == Hkv
                           else _lib.attention_gqa(q, k, vt, H, Hkv, SCALE, seq_lens=lens))
            win[split] = _lib.attention_packed_window(q, k, vt, lens, wins, H, SCALE, n_kv_heads=Hkv)
    w0 = 0
    for i, ((lo, hi), o, L) in enumerate(zip(wins, offs, lens)):
        rows = slice(w0, w0 + hi - lo)
        # split tail off: every window row is the same row of the unwindowed packed launch, bit for bit
        assert torch.equal(win[0][rows], full[0][o + lo:o + hi]), (L, lo, hi, H, Hkv)
        qh = q[o + lo:o + hi].view(hi - lo, H, 128).transpose(0, 1).float()
        kh = k[o:o + L].view(L, Hkv, 128).transpose(0, 1).float().repeat_interleave(H // Hkv, dim=0)
        vh = v[o:o + L].view(L, Hkv, 128).transpose(0, 1).float().repeat_interleave(H // Hkv, dim=0)
        ref = (torch.softmax(qh @ kh.transpose(-1, -2) * SCALE, dim=-1) @ vh).transpose(0, 1).reshape(hi - lo, d)
        for split in (0, 1):
            assert_attention_close(win[split][rows], ref, f"window [{lo},{hi}) of L={L} H={H}/{Hkv} split_tail={split}")
        w0 += hi - lo
    assert w0 == win[0].shape[0]


def test_packed_window_attention_rejects_bad_windows():
    from mmada_parallel_b200 import _lib
    q = torch.zeros(300, 512, dtype=torch.bfloat16, device="cuda")
    k, vt = q.clone(), torch.zeros(2, 4, 128, 200, dtype=torch.bfloat16, device="cuda")
    for wins in ([(0, 100), (5, 5)], [(0, 101), (0, 200)], [(-1, 10), (0, 200)]):
        with pytest.raises(_lib.MmdpError):
            _lib.attention_packed_window(q, k, vt, [100, 200], wins, 4, SCALE)


# ---------------------------------------------------------------------------------------------------------------------
# 2. forward_rows_packed(row_windows=) on tiny models
# ---------------------------------------------------------------------------------------------------------------------
_TINY = {}


def _tiny(kind):
    """bf16, fp8, or a grouped-query (4 heads, 2 kv heads) model with a q/k/v bias; max_batch 4."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    if kind not in _TINY:
        if kind == "gqa_bias":
            from oracle import llada_gqa
            cfg = llada_gqa.make_config(d_model=512, n_heads=4, n_layers=2, mlp_hidden_size=512, vocab_size=134656,
                                        max_sequence_length=512, n_kv_heads=2, include_qkv_bias=True)
            sd = llada_gqa.make_weights(cfg, seed=5)
            precision = "bf16"
        else:
            cfg, sd = tiny_cfg_and_weights(load_golden("trajectory_a_tiny.pt")["meta"])
            precision = kind
        m = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=4, precision=precision)
        m.load_state_dict(sd)
        _TINY[kind] = m
    return _TINY[kind]


def _case(lens, windows, seed):
    """Random ids per sequence and requested rows inside each window (text rows: all V columns; image rows: a column window)."""
    g = torch.Generator().manual_seed(seed)
    seqs = [torch.randint(0, 126000, (L,), generator=g).cuda() for L in lens]
    rows = []
    for L, w in zip(lens, windows):
        lo, hi = w if w is not None else (0, L)
        ra = torch.arange(lo, hi, dtype=torch.int32)[torch.randperm(hi - lo, generator=g)[: max(1, (hi - lo) // 2)].sort().values]
        rb = torch.arange(lo, hi, dtype=torch.int32)[torch.randperm(hi - lo, generator=g)[: max(1, (hi - lo) // 3)]]
        rows.append((ra.cuda(), rb.cuda()))
    return seqs, rows


def _packed(m, seqs, rows, windows):
    lens = [s.numel() for s in seqs]
    offs = [sum(lens[:j]) for j in range(len(seqs))]
    ra = torch.cat([r[0] + o for r, o in zip(rows, offs)])
    rb = torch.cat([r[1] + o for r, o in zip(rows, offs)])
    a, b = m.forward_rows_packed(torch.cat(seqs), lens, rows_a=ra, rows_b=rb, col0_b=126356, ncols_b=8192, row_windows=windows)
    res, oa, ob = [], 0, 0
    for r in rows:
        res.append((a[oa:oa + r[0].numel()], b[ob:ob + r[1].numel()]))
        oa, ob = oa + r[0].numel(), ob + r[1].numel()
    return res


@pytest.mark.parametrize("kind", ["bf16", "fp8", "gqa_bias"])
def test_forward_rows_packed_windows_tiny(kind):
    m = _tiny(kind)
    lens = [300, 77, 512, 129]
    windows = [(128, 300), None, (1, 2), (0, 129)]
    seqs, rows = _case(lens, windows, 3)
    with splits_off():
        win = _packed(m, seqs, rows, windows)
        full = _packed(m, seqs, rows, None)
        alone = [m.forward_rows(s.view(1, -1), rows_a=r[0], rows_b=r[1], col0_b=126356, ncols_b=8192, row_window=w)
                 for s, r, w in zip(seqs, rows, windows)]
    for i in range(len(lens)):
        for j in range(2):
            assert torch.equal(win[i][j], full[i][j]), (kind, i, j, "packed without windows")
            assert torch.equal(win[i][j], alone[i][j]), (kind, i, j, "own forward_rows(row_window=)")
    default = _packed(m, seqs, rows, windows)
    for i in range(len(lens)):
        for j in range(2):
            f, w = full[i][j].float(), default[i][j].float()
            dd, sc = (f - w).abs(), f.abs().max()
            assert dd.max() <= 4 * sc * 2.0 ** -8 and dd.mean() <= 0.5 * sc * 2.0 ** -8, (kind, i, j, float(dd.max()))
    m.raise_device_errors()


def test_forward_rows_packed_window_errors():
    from mmada_parallel_b200 import _lib
    m = _tiny("bf16")
    seqs, rows = _case([200, 100], [(50, 200), (0, 100)], 4)
    ids, lens = torch.cat(seqs), [200, 100]
    _lib.lib.mmdp_launch_count(1)
    for bad in ([(50, 200)], [(50, 50), None], [(0, 201), None], [(-1, 10), None]):
        with pytest.raises(ValueError):
            m.forward_rows_packed(ids, lens, rows_a=rows[0][0], row_windows=bad)
    assert _lib.lib.mmdp_launch_count(0) == 0
    # a requested row outside its sequence's window (row 10 of sequence 0, window [50, 200)) raises at the next read-back
    m.forward_rows_packed(ids, lens, rows_a=torch.tensor([60, 10], dtype=torch.int32, device="cuda"), row_windows=[(50, 200), None])
    with pytest.raises(IndexError):
        m.raise_device_errors()
    # ... and so does a row outside the packed batch; the sequence without a window takes every row
    m.forward_rows_packed(ids, lens, rows_a=torch.tensor([300], dtype=torch.int32, device="cuda"), row_windows=[(50, 200), None])
    with pytest.raises(IndexError):
        m.raise_device_errors()
    m.forward_rows_packed(ids, lens, rows_a=torch.tensor([60, 200, 299], dtype=torch.int32, device="cuda"),
                          row_windows=[(50, 200), None])
    m.raise_device_errors()


def test_forward_rows_packed_window_production_shape():
    """One block at d = 4096 / 32 heads / ff = 12288, two sequences of M's length (L = 2341 and 2329: 1024 image tokens and 256
    text positions) with M's text-step and image-step windows: bit-identical to the unwindowed packed forward and to each
    sequence's own windowed forward with the splits off, within 4 bf16 ulp of the unwindowed one with them on."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from oracle.llada import make_config
    d, ff, V = 4096, 12288, 134656
    cfg = make_config(d_model=d, n_heads=32, n_layers=1, mlp_hidden_size=ff, vocab_size=V, max_sequence_length=2432)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=2432, max_batch=2)
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*s, std):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16)
    sd = {"model.transformer.wte.weight": rnd(V, d, std=0.02), "model.transformer.ff_out.weight": rnd(V, d, std=d ** -0.5),
          "model.transformer.ln_f.weight": torch.ones(d, device="cuda", dtype=torch.bfloat16)}
    p = "model.transformer.blocks.0."
    for n, shape, std in [("q_proj", (d, d), d ** -0.5), ("k_proj", (d, d), d ** -0.5), ("v_proj", (d, d), d ** -0.5),
                          ("attn_out", (d, d), d ** -0.5), ("ff_proj", (ff, d), d ** -0.5), ("up_proj", (ff, d), d ** -0.5),
                          ("ff_out", (d, ff), ff ** -0.5)]:
        sd[p + n + ".weight"] = rnd(*shape, std=std)
    sd[p + "attn_norm.weight"] = torch.ones(d, device="cuda", dtype=torch.bfloat16)
    sd[p + "ff_norm.weight"] = torch.ones(d, device="cuda", dtype=torch.bfloat16)
    m.load_state_dict(sd)
    del sd
    lens = [2341, 2329]
    seqs = [torch.randint(0, 126000, (L,), device="cuda", generator=g) for L in lens]
    text = [(L - 256, L) for L in lens]
    image = [(L - 1281, L) for L in lens]  # (P + 1, L) with P = L - 1024 - 258
    for windows in (text, [image[0], text[1]]):
        rows = []
        for L, (lo, hi) in zip(lens, windows):
            ra = torch.arange(L - 256, L, dtype=torch.int32, device="cuda")
            rb = (torch.arange(lo, lo + 1024, dtype=torch.int32, device="cuda") if hi - lo > 256
                  else torch.arange(L - 256, L - 200, dtype=torch.int32, device="cuda"))
            rows.append((ra, rb))
        with splits_off():
            win = _packed(m, seqs, rows, windows)
            full = _packed(m, seqs, rows, None)
            for i, s in enumerate(seqs):
                alone = m.forward_rows(s.view(1, -1), rows_a=rows[i][0], rows_b=rows[i][1], col0_b=126356, ncols_b=8192,
                                       row_window=windows[i])
                for j in range(2):
                    assert torch.equal(win[i][j], full[i][j]) and torch.equal(win[i][j], alone[j]), (windows, i, j)
        default = _packed(m, seqs, rows, windows)
        for i in range(2):
            for j in range(2):
                f, w = full[i][j].float(), default[i][j].float()
                dd, sc = (f - w).abs(), f.abs().max()
                assert dd.max() <= 4 * sc * 2.0 ** -8 and dd.mean() <= 0.5 * sc * 2.0 ** -8, (windows, i, j, float(dd.max()))
        assert torch.isfinite(win[0][0].float()).all() and win[0][0].float().abs().max() > 0.1
    m.raise_device_errors()


# ---------------------------------------------------------------------------------------------------------------------
# 3. interleave_generate_batch
# ---------------------------------------------------------------------------------------------------------------------
def _m_model(max_batch, precision="bf16", max_seq_len=None):
    from mmada_parallel_b200.mmada import MMadaModelLM
    t = load_golden("trajectory_m_tiny.pt")
    cfg, sd = tiny_cfg_and_weights(t["meta"])
    cfg.mask_token_id = 126336
    m = MMadaModelLM(cfg, max_seq_len=max_seq_len or cfg.max_sequence_length, max_batch=max_batch, precision=precision)
    m.load_state_dict(sd)
    return m, t


def _m_requests(t, specs):
    """specs: (prompt length delta, text_steps, image_steps, text_cfg, image_cfg, image_temperature, seed[, n_vq])."""
    class Tok:
        bos_token_id = t["bos"]

        def __len__(self):
            return t["text_vocab_len"]

    up = SimpleNamespace(text_tokenizer=Tok())
    reqs = []
    for delta, ts, ims, tcfg, icfg, itemp, seed, *n_vq in specs:
        conf = SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=n_vq[0] if n_vq else t["num_vq_tokens"],
                                                                           codebook_size=8192)),
                               dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=t["max_seq_length"])))
        g = torch.Generator().manual_seed(1000 + seed)
        inp, unc = t["input_ids"], t["uncond_input_ids"]
        if delta >= 0:
            extra = torch.randint(0, 126000, (delta,), generator=g)
            inp, unc = torch.cat([inp[:1], extra, inp[1:]]), torch.cat([unc[:1], extra, unc[1:]])
        else:
            inp, unc = torch.cat([inp[:1], inp[1 - delta:]]), torch.cat([unc[:1], unc[1 - delta:]])
        reqs.append(dict(input_ids=inp, uncond_input_ids=unc, reserved_token_mapping={"<|soi|>": t["soi"], "<|eoi|>": t["eoi"]},
                         config=conf, uni_prompting=up, text_steps=ts, image_steps=ims, text_cfg=tcfg, image_cfg=icfg,
                         image_temperature=itemp, _seed=seed))
    return reqs


def _run_m(model, reqs):
    """(sequential results, generator states), (batch results, generator states) on fresh generators."""
    from mmada_parallel_b200.generators.batch import interleave_generate_batch
    out = []
    for batched in (False, True):
        rs = [dict({k: v for k, v in r.items() if k != "_seed"}, generator=torch.Generator().manual_seed(r["_seed"])) for r in reqs]
        res = interleave_generate_batch(model, rs) if batched else [model.interleave_generate(**r) for r in rs]
        out.append(([(a.cpu(), b.cpu()) for a, b in res], [r["generator"].get_state() for r in rs]))
    return out


def _assert_same_m(seq, bat, what):
    assert len(seq[0]) == len(bat[0])
    for i, ((ia, ta), (ib, tb)) in enumerate(zip(seq[0], bat[0])):
        assert ia.shape == ib.shape and torch.equal(ia, ib), (what, "image ids", i)
        assert ta.shape == tb.shape and torch.equal(ta, tb), (what, "text ids", i)
    for i, (ga, gb) in enumerate(zip(seq[1], bat[1])):
        assert torch.equal(ga, gb), (what, "generator state", i)


_SPECS = [(0, 8, 4, 2.5, 4.0, 1.0, 42), (7, 6, 6, 0.0, 3.5, 0.5, 5), (-5, 10, 3, 1.5, 2.0, 2.0, 7)]


@pytest.mark.parametrize("n", [1, 2, 3])
def test_interleave_generate_batch_equals_sequential_calls(n):
    """1, 2 and 3 requests with different prompt lengths, text / image steps, CFG scales and image temperatures: with the splits
    off, every returned tensor and every generator state equals sequential interleave_generate calls, once with all 2N
    sequences in one packed forward and once with max_batch = 2 (one request per packed forward)."""
    for max_batch in (2 * n, 2):
        model, t = _m_model(max_batch)
        with splits_off():
            seq, bat = _run_m(model, _m_requests(t, _SPECS[:n]))
        _assert_same_m(seq, bat, (n, max_batch))


def test_interleave_generate_batch_fp8():
    model, t = _m_model(6, precision="fp8")
    with splits_off():
        seq, bat = _run_m(model, _m_requests(t, _SPECS))
    _assert_same_m(seq, bat, "fp8")


def test_interleave_generate_batch_with_row_windows():
    """Sequences of L >= 1024 (1024 image tokens) take interleave_generate's last-block row windows (text rows on text steps,
    from the image rows on image steps), in the batch per sequence: still equal to sequential calls, and with 3 packed forwards
    per step on max_batch = 2 next to a short request without windows."""
    model, t = _m_model(4, max_seq_len=1100)
    specs = [(0, 6, 3, 2.5, 4.0, 1.0, 11, 1024), (9, 5, 2, 0.0, 3.5, 1.0, 12, 1024), (3, 4, 2, 1.0, 2.0, 1.0, 13)]
    with splits_off():
        seq, bat = _run_m(model, _m_requests(t, specs))
    _assert_same_m(seq, bat, "windows")
    model2, _ = _m_model(2, max_seq_len=1100)
    with splits_off():
        seq2, bat2 = _run_m(model2, _m_requests(t, specs))
    _assert_same_m(seq2, bat2, "windows, max_batch 2")
    _assert_same_m(seq, seq2, "same model, other max_batch")
