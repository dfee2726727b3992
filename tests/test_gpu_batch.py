"""Packed variable-length batches on the H100: the packed attention kernel, the V^T pad rule, `forward_rows_packed` (bf16 and
FP8, tiny and production shapes) and `generate_ti2ti_batch` against sequential `generate_ti2ti` calls and the real reference."""
import contextlib
import io
import math

import pytest
import torch

from helpers import load_golden, tiny_cfg_and_weights, tiny_gpu_model
from test_gpu_kernels import assert_attention_close, attn_version  # noqa: F401  (attn_version: the kernel-generation fixture)

pytestmark = pytest.mark.gpu

MASK, NEW_LINE = 126336, 126084


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


@contextlib.contextmanager
def splits_off():
    """GEMM split-K tail and attention KV-split tail off: which tiles they touch depends on the problem size, so only without
    them is a packed row bit-identical to the same row computed alone."""
    from mmada_parallel_b200 import _lib
    _lib.lib.mmdp_set_gemm_splitk(0)
    _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 0))
    try:
        yield
    finally:
        _lib.lib.mmdp_set_gemm_splitk(2)
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))


# ---------------------------------------------------------------------------------------------------------------------
# 1. packed attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [2, 4])  # 68 query tiles: no split; 136 tiles on 132 SMs: the last 4 (of the 2414 sequence) split
def test_packed_attention(H, attn_version):
    from mmada_parallel_b200 import _lib
    lens = [1, 63, 64, 127, 128, 129, 1000, 2414]
    d, M, n = H * 128, sum(lens), len(lens)
    Lpad = (max(lens) + 7) // 8 * 8
    torch.manual_seed(7 + H)
    q = torch.randn(M, d, device="cuda").to(torch.bfloat16)
    k = torch.randn(M, d, device="cuda").to(torch.bfloat16)
    v = torch.randn(M, d, device="cuda").to(torch.bfloat16)
    vt = torch.zeros(n, H, 128, Lpad, dtype=torch.bfloat16, device="cuda")
    offs = [sum(lens[:i]) for i in range(n)]
    for i, (o, L) in enumerate(zip(offs, lens)):
        vt[i, :, :, :L] = v[o:o + L].view(L, H, 128).permute(1, 2, 0)
    scale = 1.0 / math.sqrt(128.0)
    out = {}
    try:
        for split in (1, 0):
            _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", split))
            out[split] = _lib.attention_packed(q, k, vt, lens, H, scale)
        # split tail off: each sequence bit-identical to its own mmdp_attention call
        for i, (o, L) in enumerate(zip(offs, lens)):
            Lp = (L + 7) // 8 * 8
            alone = _lib.attention(q[o:o + L].contiguous(), k[o:o + L].contiguous(), vt[i:i + 1, :, :, :Lp].contiguous(), 1, H, L, scale)
            assert torch.equal(out[0][o:o + L], alone), (L, H)
    finally:
        _lib.check(_lib.lib.mmdp_set_option(b"attn_split_tail", 1))
    for i, (o, L) in enumerate(zip(offs, lens)):
        qh, kh, vh = (t[o:o + L].view(L, H, 128).transpose(0, 1).float() for t in (q, k, v))
        ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(0, 1).reshape(L, d)
        for split in (1, 0):
            assert_attention_close(out[split][o:o + L], ref, f"packed attention L={L} H={H} split_tail={split}")
    assert (out[0].float() - out[1].float()).abs().max().item() <= 2.0 ** -8 * max(o.abs().max().item() for o in out.values())


# ---------------------------------------------------------------------------------------------------------------------
# 2.-3. forward_rows_packed on the tiny model
# ---------------------------------------------------------------------------------------------------------------------
def _tiny(precision="bf16", max_batch=4):
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    meta = load_golden("trajectory_a_tiny.pt")["meta"]
    cfg, sd = tiny_cfg_and_weights(meta)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=max_batch, precision=precision)
    m.load_state_dict(sd)
    return m


def _seqs(lens, seed, vocab=134656):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (L,), generator=g).cuda() for L in lens]


def _rows(L, seed):
    g = torch.Generator().manual_seed(seed)
    ra = torch.randperm(L, generator=g)[: max(1, L // 3)].sort().values
    rb = torch.randperm(L, generator=g)[: max(1, L // 4)]
    return ra.to(torch.int32).cuda(), rb.to(torch.int32).cuda()


def _packed(m, seqs, rows, order):
    """forward_rows_packed over seqs in `order`; returns per sequence (text logits, image logits) in the original indexing."""
    lens = [seqs[i].numel() for i in order]
    offs = [sum(lens[:j]) for j in range(len(order))]
    ra = torch.cat([rows[i][0] + o for i, o in zip(order, offs)])
    rb = torch.cat([rows[i][1] + o for i, o in zip(order, offs)])
    a, b = m.forward_rows_packed(torch.cat([seqs[i] for i in order]), lens, rows_a=ra, rows_b=rb, col0_b=126356, ncols_b=8192)
    res, oa, ob = {}, 0, 0
    for i in order:
        na, nb = rows[i][0].numel(), rows[i][1].numel()
        res[i] = (a[oa:oa + na], b[ob:ob + nb])
        oa, ob = oa + na, ob + nb
    return res


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_forward_rows_packed_tiny(precision):
    m = _tiny(precision)
    lens = [300, 77, 512, 129]
    seqs = _seqs(lens, 11)
    rows = [_rows(L, 20 + i) for i, L in enumerate(lens)]
    alone = {}
    with splits_off():
        for i, s in enumerate(seqs):
            alone[i] = m.forward_rows(s.view(1, -1), rows_a=rows[i][0], rows_b=rows[i][1], col0_b=126356, ncols_b=8192)
        packed = _packed(m, seqs, rows, [0, 1, 2, 3])
        reordered = _packed(m, seqs, rows, [2, 0, 3, 1])
    for i in range(len(lens)):
        for j in range(2):
            assert torch.equal(packed[i][j], alone[i][j]), (precision, lens[i], j)
            assert torch.equal(reordered[i][j], packed[i][j]), (precision, lens[i], j, "reordered")
    default = _packed(m, seqs, rows, [0, 1, 2, 3])
    for i in range(len(lens)):
        for j in range(2):
            f, w = alone[i][j].float(), default[i][j].float()
            dd, sc = (f - w).abs(), f.abs().max()
            assert dd.max() <= 4 * sc * 2.0 ** -8 and dd.mean() <= 0.5 * sc * 2.0 ** -8, (precision, lens[i], float(dd.max()))
    m.raise_device_errors()


def test_vt_pad_rule_across_packed_and_ordinary_forwards():
    """Columns [L_s, Lpad) of every V^T block a forward reads must be zero. A packed forward with short sequences right after one
    with long sequences (same padded stride), and an ordinary forward after packed ones, give the bits of a fresh context."""
    m = _tiny(max_batch=4)
    long_seqs, short_seqs = _seqs([200, 198, 197], 3), _seqs([130, 199, 140], 4)
    rows_l = [_rows(s.numel(), 40 + i) for i, s in enumerate(long_seqs)]
    rows_s = [_rows(s.numel(), 50 + i) for i, s in enumerate(short_seqs)]
    one = _seqs([150], 5)[0].view(1, -1)
    r1 = _rows(150, 60)
    _packed(m, long_seqs, rows_l, [0, 1, 2])
    after_long = _packed(m, short_seqs, rows_s, [0, 1, 2])
    ordinary_after = m.forward_rows(one, rows_a=r1[0], rows_b=r1[1], col0_b=126356, ncols_b=8192)
    fresh = _tiny(max_batch=4)
    want = _packed(fresh, short_seqs, rows_s, [0, 1, 2])
    fresh2 = _tiny(max_batch=4)
    want1 = fresh2.forward_rows(one, rows_a=r1[0], rows_b=r1[1], col0_b=126356, ncols_b=8192)
    for i in range(3):
        assert torch.equal(after_long[i][0], want[i][0]) and torch.equal(after_long[i][1], want[i][1]), i
    assert torch.equal(ordinary_after[0], want1[0]) and torch.equal(ordinary_after[1], want1[1])


# ---------------------------------------------------------------------------------------------------------------------
# 4. production shapes
# ---------------------------------------------------------------------------------------------------------------------
def test_forward_rows_packed_production_shapes():
    """Two blocks at d = 4096 / 32 heads / ff = 12288, sequences [2414, 1313, 700] in one packed forward: bit-identical to three
    B = 1 forwards with the splits off."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from oracle.llada import make_config
    d, ff, V, nl = 4096, 12288, 134656, 2
    cfg = make_config(d_model=d, n_heads=32, n_layers=nl, mlp_hidden_size=ff, vocab_size=V, max_sequence_length=2432)
    m = LLaDAForMultiModalGeneration(cfg, max_seq_len=2432, max_batch=3)
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*s, std):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16)
    sd = {"model.transformer.wte.weight": rnd(V, d, std=0.02), "model.transformer.ff_out.weight": rnd(V, d, std=d ** -0.5),
          "model.transformer.ln_f.weight": torch.ones(d, device="cuda", dtype=torch.bfloat16)}
    for li in range(nl):
        p = f"model.transformer.blocks.{li}."
        for n, shape, std in [("q_proj", (d, d), d ** -0.5), ("k_proj", (d, d), d ** -0.5), ("v_proj", (d, d), d ** -0.5),
                              ("attn_out", (d, d), d ** -0.5), ("ff_proj", (ff, d), d ** -0.5), ("up_proj", (ff, d), d ** -0.5),
                              ("ff_out", (d, ff), ff ** -0.5)]:
            sd[p + n + ".weight"] = rnd(*shape, std=std)
        sd[p + "attn_norm.weight"] = torch.ones(d, device="cuda", dtype=torch.bfloat16)
        sd[p + "ff_norm.weight"] = torch.ones(d, device="cuda", dtype=torch.bfloat16)
    m.load_state_dict(sd)
    del sd
    lens = [2414, 1313, 700]
    seqs = _seqs(lens, 8, vocab=126000)
    rows = []
    for L in lens:
        rows.append((torch.arange(L - 256, L, dtype=torch.int32, device="cuda"),
                     torch.arange(0, L - 256, 3, dtype=torch.int32, device="cuda")[:1024]))
    with splits_off():
        packed = _packed(m, seqs, rows, [0, 1, 2])
        for i, s in enumerate(seqs):
            a, b = m.forward_rows(s.view(1, -1), rows_a=rows[i][0], rows_b=rows[i][1], col0_b=126356, ncols_b=8192)
            assert torch.equal(packed[i][0], a) and torch.equal(packed[i][1], b), lens[i]
    assert torch.isfinite(packed[0][0].float()).all() and packed[0][0].float().abs().max() > 0.1
    m.raise_device_errors()


# ---------------------------------------------------------------------------------------------------------------------
# 5.-6. the batch loop
# ---------------------------------------------------------------------------------------------------------------------
def _layout(lay, prompt_delta, h, w, seed):
    """A request layout derived from a fixture layout (image region, then text region): the prompt before the image region
    grows or shrinks by prompt_delta tokens, the image grid becomes h x w (newline after every row)."""
    ids = lay["input_ids"][0].tolist()
    img0 = lay["image_start"]
    img_len = lay["seq_len"] + lay["seq_len"] // lay["newline_every"]
    pre, post = ids[:img0], ids[img0 + img_len:]
    g = torch.Generator().manual_seed(seed)
    if prompt_delta >= 0:
        pre = pre[:1] + torch.randint(0, 126000, (prompt_delta,), generator=g).tolist() + pre[1:]
    else:
        pre = pre[:1] + pre[1 - prompt_delta:]
    region = ([MASK] * w + [NEW_LINE]) * h
    n_text = lay["text_end"] - lay["text_start"]
    text_start = len(pre) + len(region) + (lay["text_start"] - (img0 + img_len))
    return dict(input_ids=torch.tensor([pre + region + post], dtype=torch.int64), text_start=text_start,
                text_end=text_start + n_text, image_start=len(pre), seq_len=h * w, newline_every=w,
                uncon_text=lay["uncon_text"], uncon_image=lay["uncon_image"])


def _run_both(model, reqs, global_seed=999):
    """(sequential results, traces, generator states), (batch results, traces, generator states) on fresh generators."""
    from mmada_parallel_b200.generators.batch import generate_ti2ti_batch
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    out = []
    for batched in (False, True):
        rs = [dict(r, generator=torch.Generator().manual_seed(r["_seed"]), _trace=[]) for r in reqs]
        for r in rs:
            r.pop("_seed")
        torch.manual_seed(global_seed)
        with quiet():
            res = generate_ti2ti_batch(model, rs) if batched else [generate_ti2ti(model, **r) for r in rs]
        out.append((res, [r["_trace"] for r in rs], [r["generator"].get_state() for r in rs]))
    return out


def _assert_same(seq, bat):
    for i, (a, b) in enumerate(zip(seq[0], bat[0])):
        assert a == b, ("results", i)
    for i, (ta, tb) in enumerate(zip(seq[1], bat[1])):
        assert len(ta) == len(tb), ("trace length", i)
        for sa, sb in zip(ta, tb):
            assert sa.keys() == sb.keys() and sa["step"] == sb["step"]
            for k in sa:
                if k != "step":
                    assert torch.equal(sa[k], sb[k]), ("trace", i, sa["step"], k)
    for i, (ga, gb) in enumerate(zip(seq[2], bat[2])):
        assert torch.equal(ga, gb), ("generator state", i)


def test_batch_loop_equals_sequential_calls():
    """Different prompt lengths, square and non-square grids, different text_steps / timesteps, greedy, temperature 1, and both
    CFGs with text Gumbel: per-step traces, final ids, text and generator states equal sequential calls (splits off). The
    second batch has 4 requests with both CFGs on a max_batch = 3 model: 8 unconditional sequences run as 3 packed forwards."""
    t = load_golden("trajectory_a_tiny.pt")
    lay = t["layout"]
    kw = {r["name"]: dict(r["kwargs"]) for r in t["runs"]}
    model, _, _ = tiny_gpu_model(t["meta"], max_batch=3)
    reqs = [dict(_layout(lay, 0, 4, 4, 1), **dict(kw["greedy_cfgimg4"], text_steps=8, timesteps=4), _seed=42),
            dict(_layout(lay, 9, 3, 5, 2), **dict(kw["canonical_temp1"], text_steps=6, timesteps=3), _seed=43),
            dict(_layout(lay, -7, 5, 4, 3), **dict(kw["both_cfg_texttemp"], text_steps=10, timesteps=5), _seed=44),
            dict(_layout(lay, 23, 2, 6, 4), **dict(kw["no_cfg"], text_steps=5, timesteps=2), _seed=45)]
    with splits_off():
        seq, bat = _run_both(model, reqs)
    _assert_same(seq, bat)
    many = [dict(_layout(lay, d, h, w, 10 + i), **dict(kw["both_cfg_texttemp"], text_steps=ts, timesteps=tm), _seed=60 + i)
            for i, (d, h, w, ts, tm) in enumerate([(0, 4, 4, 8, 4), (5, 3, 4, 7, 4), (-4, 4, 3, 9, 3), (13, 2, 2, 6, 6)])]
    with splits_off():
        seq, bat = _run_both(model, many)
    _assert_same(seq, bat)


def test_batch_against_real_reference_separated():
    """The fixture runs of the REAL reference (trajectory_a_separated.pt), each packed next to two other requests of different
    lengths, with default options: the request's ids equal the reference's after every step."""
    from mmada_parallel_b200.generators.batch import generate_ti2ti_batch
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    from oracle import llada
    from oracle.make_golden_separated import separated_weights
    t = load_golden("trajectory_a_separated.pt")
    cfg = llada.make_config(**t["meta"]["tiny"])
    lay = t["layout"]
    base = {k: lay[k] for k in ("input_ids", "text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text",
                                "uncon_image")}
    for run in t["runs"]:
        sd, _ = separated_weights(cfg, run["weight_seed"])
        model = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=3)
        model.load_state_dict(sd)
        tr = []
        # the fixture request first: still-masked image tokens come from the global CPU RNG after the loop, in request order
        reqs = [dict(base, **run["kwargs"], generator=torch.Generator().manual_seed(run["seed"]), _trace=tr),
                dict(_layout(lay, 11, 4, 4, 1), **run["kwargs"], generator=torch.Generator().manual_seed(1)),
                dict(_layout(lay, -3, 2, 5, 2), **run["kwargs"], generator=torch.Generator().manual_seed(2))]
        torch.manual_seed(run["global_seed"])
        res = generate_ti2ti_batch(model, reqs)
        for step, rec in enumerate(tr):
            assert torch.equal(rec["ids_after_text"].cpu(), run["ids_after_text"][step]), (run["name"], step, "text step")
            if "ids_after_image" in rec:
                assert torch.equal(rec["ids_after_image"].cpu(), run["ids_after_image"][step]), (run["name"], step, "image step")
        assert res[0][1] == run["text_tokens"] and res[0][0] == run["image_tokens"], run["name"]
        del model


# ---------------------------------------------------------------------------------------------------------------------
# 7. errors
# ---------------------------------------------------------------------------------------------------------------------
def test_batch_errors():
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.generators.batch import generate_ti2ti_batch
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    t = load_golden("trajectory_a_tiny.pt")
    lay = t["layout"]
    model, cfg, _ = tiny_gpu_model(t["meta"], max_batch=3)
    kw = dict(t["runs"][0]["kwargs"], text_steps=2, timesteps=1)
    good = dict(_layout(lay, 0, 4, 4, 1), **kw)
    bad = dict(_layout(lay, 5, 4, 4, 2), **kw)
    bad["input_ids"] = bad["input_ids"].clone()
    bad["input_ids"][0, 0] = cfg.vocab_size + 5
    with pytest.raises(IndexError), quiet():
        generate_ti2ti_batch(model, [dict(good, generator=torch.Generator()), dict(bad, generator=torch.Generator())])
    model.raise_device_errors()  # cleared by the read above
    # capacity: checked before anything is launched
    too_long = dict(_layout(lay, cfg.max_sequence_length, 4, 4, 3), **kw)
    _lib.lib.mmdp_launch_count(1)
    with pytest.raises(ValueError):
        generate_ti2ti_batch(model, [dict(good, generator=torch.Generator()), dict(too_long, generator=torch.Generator())])
    with pytest.raises(ValueError):
        model.forward_rows_packed(torch.zeros(40, dtype=torch.int64, device="cuda"), [10, 10, 10, 10])
    with pytest.raises(ValueError):
        model.forward_rows_packed(torch.zeros(600, dtype=torch.int64, device="cuda"), [600])
    assert _lib.lib.mmdp_launch_count(0) == 0
    # the tensor-parallel model has no packed forward
    with pytest.raises(TypeError):
        generate_ti2ti_batch(object.__new__(TensorParallelLLaDA), [dict(good, generator=torch.Generator())])
