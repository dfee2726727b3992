"""The oracle (CPU restatement) against the golden vectors produced by the REAL reference (oracle/make_golden.py)."""
import pytest
import torch

from helpers import load_golden, tiny_cfg_and_weights
from oracle import generate as G
from oracle import llada
from oracle import sampling as S


@pytest.fixture(scope="module")
def tiny():
    g = load_golden("forward_tiny.pt")
    cfg, sd = tiny_cfg_and_weights(g["meta"])
    return g, cfg, sd, llada.OracleModel(cfg, sd)


def sort_order_matches_fixture(kat):
    p = kat["sort_probe"]
    return torch.equal(torch.sort(p["x"], dim=-1, descending=False).indices, p["idx"])


def test_forward_matches_reference_logits(tiny):
    g, cfg, sd, model = tiny
    lo = model(g["ids"]).logits
    assert torch.equal(lo[0][:, g["cols"]], g["logits_cols"])
    assert torch.equal(lo[0].argmax(-1), g["argmax"])
    lo2 = model(g["ids2"]).logits
    assert torch.equal(lo2[:, :, g["cols"]], g["logits2_cols"])
    # batch rows are independent: row 0 of the B=2 forward equals the B=1 forward
    assert torch.equal(lo2[0], lo[0])


def test_sampler_known_answers():
    kat = load_golden("sampler_kat.pt")
    same_sort = sort_order_matches_fixture(kat)
    for c in kat["a_mask_by_random_topk"]:
        m, conf = S.mask_by_random_topk_a(c["k"], c["probs"], c["temp"], c["noise"])
        if same_sort:
            assert torch.equal(m, c["masking"])
        # tie-independent properties hold for any sort order, and for the stable rule the kernel uses
        for mm in (m, S.mask_by_random_topk_a(c["k"], c["probs"], c["temp"], c["noise"], stable=True)[0], c["masking"]):
            k = min(max(c["k"], 0), c["probs"].numel() - 1)
            assert int(mm.sum()) == k
            if 0 < k:
                assert conf[mm].float().max() <= conf[~mm].float().min()
    for c in kat["a_add_gumbel_noise"]:
        out = S.add_gumbel_noise_a(c["logits"], c["temp"], c["uniform"])
        assert torch.equal(out, c["out"]) and torch.equal(out.argmax(-1), c["argmax"])
    for (n, steps), want in kat["a_num_transfer"].items():
        assert S.get_num_transfer_tokens_a(n, steps) == want
    assert [S.sched_len(1024, s, 128) for s in range(128)] == kat["a_sched_len_1024_128"]
    assert kat["a_sched_len_1024_128"][-1] == -1  # fp32 cos(pi/2) < 0: one token always stays masked
    for c in kat["m_mask_by_random_topk"]:
        m, _ = S.mask_by_random_topk_m(c["k"], c["probs"], c["temp"], c["noise"])
        assert torch.equal(m, c["masking"])
    for (n, steps), want in kat["m_num_transfer"].items():
        assert S.get_num_transfer_tokens_m(n, steps) == want
    assert torch.equal(S.lfq_codebook_entry(kat["m_lfq"]["idx"], 13), kat["m_lfq"]["zq"])


def test_trajectories_a(tiny):
    _, cfg, sd, model = tiny
    t = load_golden("trajectory_a_tiny.pt")
    same_sort = sort_order_matches_fixture(load_golden("sampler_kat.pt"))
    lay = t["layout"]
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    for run in t["runs"]:
        torch.manual_seed(run["global_seed"])
        img, txt = G.generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                    **args, **run["kwargs"])
        assert txt == run["text_tokens"], run["name"]
        if same_sort:
            assert img == run["image_tokens"], run["name"]
        assert len(img) == lay["seq_len"] and all(0 <= v < 8192 for v in img)
    # the caller's tensor is never modified (:140)
    before = lay["input_ids"].clone()
    G.generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(0), **args, **t["runs"][0]["kwargs"])
    assert torch.equal(before, lay["input_ids"])


def test_trajectories_m(tiny):
    _, cfg, sd, model = tiny
    t = load_golden("trajectory_m_tiny.pt")
    for run in t["runs"]:
        img, txt = G.interleave_generate(model, t["input_ids"], t["uncond_input_ids"], soi_id=t["soi"], eoi_id=t["eoi"],
                                         bos_id=t["bos"], mask_id=t["mask_id"], num_vq_tokens=t["num_vq_tokens"],
                                         codebook_size=8192, max_seq_length=t["max_seq_length"],
                                         text_vocab_len=t["text_vocab_len"],
                                         generator=torch.Generator().manual_seed(run["seed"]), **run["kwargs"])
        assert torch.equal(img, run["image_ids"]) and torch.equal(txt, run["text_ids"]), run["name"]
    with pytest.raises(ValueError):
        G.interleave_generate(model, t["input_ids"], t["uncond_input_ids"], 0.0, 0.0, 4, 2, 1, 2, 3, 126336, 16, 8192, 12, 126349)


def test_edge_cases():
    # empty / fully un-masked text span: nothing changes
    ids = torch.tensor([5, 6, 7])
    logits = torch.randn(3, 64).to(torch.bfloat16)
    new, _, _ = S.text_step(logits, ids, 126336, 2)
    assert torch.equal(new, ids)
    # k larger than the number of masked positions: only masked positions change
    ids = torch.tensor([126336, 6, 126336])
    new, x0, _ = S.text_step(logits, ids, 126336, 3)
    assert new[1] == 6 and new[0] == x0[0] and new[2] == x0[2]
    # first-index tie rule of argmax on bf16 logits
    l = torch.zeros(1, 32, dtype=torch.bfloat16)
    l[0, 7] = l[0, 19] = 1.0
    _, x0, _ = S.text_step(l, torch.tensor([126336]), 126336, 1)
    assert int(x0[0]) == 7
    # image step with a single unknown token: mask_len clamps to 1 and one token stays masked (Appendix A5)
    cond = torch.randn(8, 8192).to(torch.bfloat16)
    vq = torch.arange(8)
    vq[3] = -1
    out = S.image_step("A", cond, None, None, 0.0, 0.0, vq, 126336, 0, 0.0, None, torch.zeros(8, dtype=torch.bfloat16), 8192)
    assert out["mask_len"] == 1 and int(out["masking"].sum()) == 1 and bool(out["masking"][3])


def test_magvit_decoder_matches_reference_golden():
    from oracle import magvit as OM
    g = load_golden("magvit_decode.pt")["small"]
    cfg = OM.decoder_config(**g["cfg"])
    w = OM.make_weights(cfg, g["weight_seed"])
    out = OM.decode_code(g["idx"], w, cfg)
    assert tuple(out.shape) == tuple(g["shape"])
    assert torch.equal(out[:, :, ::g["stride"], ::g["stride"]], g["image"])
    names = OM.param_shapes(OM.decoder_config())
    assert sum(torch.Size(s).numel() for s in names.values()) > 39_000_000  # the real decoder (~39.9 M parameters)


def test_magvit_encoder_matches_reference_golden():
    from oracle import magvit as OM
    g = load_golden("magvit_encode.pt")["small"]
    cfg = OM.encoder_config(**g["cfg"])
    w = OM.make_encoder_weights(cfg, g["weight_seed"])
    px = torch.rand(g["batch"], 3, g["res"], g["res"], generator=torch.Generator().manual_seed(g["pixel_seed"])) * 2 - 1
    assert torch.equal(OM.encoder_forward(px, w, cfg), g["z"])
    assert torch.equal(OM.get_code(px, w, cfg), g["ids"])
    # decode(get_code(x)) round trip stays on the code grid: ids -> +-1 bits -> ids (idempotence of the LFQ codebook)
    from oracle.sampling import lfq_codebook_entry
    ids = g["ids"]
    side = int(ids.shape[1] ** 0.5)
    assert torch.equal(OM.lfq_indices(lfq_codebook_entry(ids, 13).view(ids.shape[0], 13, side, side), 13), ids)


def test_stepwise_preview_loop_matches_reference_golden(tiny):
    """oracle.generate.generate_ti2ti_stepwise == the reference's Gradio preview loop (A/app.py:143-398): every yielded
    (step, text, status), the ids handed to the VQ decoder and the greyed-out cells (fixture made by
    oracle/make_golden_stepwise.py from the real reference)."""
    t = load_golden("trajectory_stepwise_tiny.pt")
    model = tiny[3]
    same_sort = sort_order_matches_fixture(load_golden("sampler_kat.pt"))  # tie order of torch.sort on this machine
    lay = t["layout"]
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    for run in t["runs"]:
        decoded = []

        def preview(sampled, masking, masked_idx):
            decoded.append(sampled.clone())
            return masking.nonzero().flatten().tolist() if masking is not None else list(masked_idx)

        ys = list(G.generate_ti2ti_stepwise(model, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                            tokenizer=G.PieceTokenizer(), preview=preview, **args, **run["kwargs"]))
        assert [s for s, _, _, _ in ys] == [y[0] for y in run["yields"]], run["name"]
        assert len(decoded) == len(run["decoded"])
        if same_sort:
            assert [(s, txt, st, im is not None) for s, txt, im, st in ys] == [tuple(y) for y in run["yields"]], run["name"]
            assert [im for _, _, im, _ in ys] == run["overlays"], run["name"]
            assert all(torch.equal(a, b) for a, b in zip(decoded, run["decoded"]))


def test_mmu_generate_matches_reference_golden(tiny):
    """oracle.generate.mmu_generate == MMadaModelLM.mmu_generate (M/models/modeling_mmada.py:619-691) on the tiny model:
    B=1 two blocks, B=2 with CFG, uneven per-step counts, all-ones attention mask (oracle/make_golden_mmu.py)."""
    t = load_golden("trajectory_mmu_tiny.pt")
    model = tiny[3]
    for run in t["runs"]:
        am = torch.ones_like(run["out"]) if run["ones_mask"] else None
        out = G.mmu_generate(model, run["idx"], attention_mask=am, **run["kwargs"])
        assert torch.equal(out, run["out"]), run["name"]
    with pytest.raises(NotImplementedError):
        G.mmu_generate(model, t["runs"][0]["idx"], remasking="random")
    # (temperature > 0 and zero-containing attention masks: test_variant_m_modes_match_reference_golden)


def test_generate_image_t2i_matches_reference_golden(tiny):
    """oracle.generate.generate_image == A/generators/image_generation_generator.py::generate_image (MaskGit T2I decoding,
    use_cache=False) on the tiny model: greedy, temperature 1, CFG 3, and an 18-step run that exits early
    (oracle/make_golden_t2i.py). Groundwork for the product path (DESIGN.md section 6)."""
    t = load_golden("trajectory_t2i_tiny.pt")
    model, lay = tiny[3], t["layout"]
    for run in t["runs"]:
        tr = []
        out = G.generate_image(model, lay["prompt"], generator=torch.Generator().manual_seed(run["seed"]), seq_len=lay["seq_len"],
                               newline_every=lay["newline_every"], code_start=lay["code_start"], uncon_ids=lay["uncon_ids"],
                               text_vocab_size=126356, codebook_size=8192, trace=tr, **run["kwargs"])
        assert torch.equal(out, run["vq_ids"]), run["name"]
        assert len(tr) == run["steps_run"] and out.shape == (1, lay["seq_len"])
        assert int((out < 126356).sum()) == 0 and int((out >= 126356 + 8192).sum()) == 0


def test_variant_m_modes_match_reference_golden(tiny):
    """t2i_generate, mmu_generate (zero-containing attention mask; temperature > 0) and interleave_generate with
    text_temperature > 0 against the ids the REAL MMadaModelLM produced (oracle/make_golden_m_modes.py)."""
    _, cfg, sd, model = tiny
    t = load_golden("trajectory_m_modes_tiny.pt")
    tv = t["meta"]["text_vocab_len"]
    for r in t["t2i"]:
        ids = r["input_ids"].clone()
        out = G.t2i_generate(model, ids, r["uncond_input_ids"].clone(), attention_mask=r["attention_mask"],
                             uncond_attention_mask=r["attention_mask"], generator=torch.Generator().manual_seed(r["seed"]),
                             text_vocab_len=tv, **r["kwargs"])
        assert torch.equal(out, r["sampled"]) and torch.equal(ids, r["final_input_ids"]), r["name"]
    for r in t["mmu"]:
        if r["global_seed"] is not None:
            torch.manual_seed(r["global_seed"])
        assert torch.equal(G.mmu_generate(model, r["idx"], attention_mask=r["attention_mask"], **r["kwargs"]), r["out"]), r["name"]
    for r in t["interleave"]:
        torch.manual_seed(r["global_seed"])
        img, txt = G.interleave_generate(model, r["input_ids"], r["uncond_input_ids"], soi_id=126085, eoi_id=126086, bos_id=126080,
                                         mask_id=126336, num_vq_tokens=16, codebook_size=8192, max_seq_length=12, text_vocab_len=tv,
                                         generator=torch.Generator().manual_seed(r["seed"]), **r["kwargs"])
        assert torch.equal(img, r["image_ids"]) and torch.equal(txt, r["text_ids"]), r["name"]


def test_separated_model_trajectories_match_reference_golden():
    """The "well-separated" tiny model (oracle/make_golden_separated.py): the oracle reproduces the REAL reference's per-step ids
    on all three configurations (greedy / bench-like / both CFGs + text Gumbel) - the fixture the H100 path must match bit for
    bit in tests/test_gpu_model.py::test_trajectory_bit_equal_to_reference_on_separated_model."""
    from oracle.make_golden_separated import separated_weights, trajectory
    t = load_golden("trajectory_a_separated.pt")
    cfg = llada.make_config(**t["meta"]["tiny"])
    for run in t["runs"]:
        sd, _ = separated_weights(cfg, run["weight_seed"])
        img, txt, tr = trajectory(llada.OracleModel(cfg, sd), t["layout"], run["kwargs"], run["seed"], run["global_seed"])
        assert img == run["image_tokens"] and txt == run["text_tokens"], run["name"]
        for step, rec in enumerate(tr):
            assert torch.equal(rec["ids_after_text"], run["ids_after_text"][step])


def test_token_cache_forward_matches_reference_golden(tiny):
    """oracle.llada.CachedOracleModel == the reference's LLaDAModelLM.forward(use_cache=True, to_compute_mask, cat) after
    caching(True) (modeling_llada.py:929-940, :1244-1245, :1406-1413): one full forward and three partial ones per cache key
    (oracle/make_golden_cache.py)."""
    _, cfg, sd, _ = tiny
    t = load_golden("token_cache_tiny.pt")
    om = llada.CachedOracleModel(cfg, sd)
    for case in t["cases"]:
        for st in case["steps"]:
            lg = om(st["ids"], to_compute_mask=st["mask"], cat=case["cat"]).logits
            assert torch.equal(lg[:, :, st["cols"]], st["logits_cols"]), case["name"]
            assert torch.equal(lg.float().argmax(-1), st["argmax"])
