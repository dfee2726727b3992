"""Adjacent generation modes of SURVEY.md section 8f rank 3 on the H100, each in lock-step with the oracle running on the
SAME (GPU-computed) logits and the same replayed noise - integer outputs must be equal at every step:
  A  generate_image        (generators/image_generation_generator.py:15-251, MaskGit text-to-image)
  M  t2i_generate          (models/modeling_mmada.py:265-359)
  M  interleave_generate / mmu_generate with a text temperature > 0 (fp64 Gumbel-max, :49-60) and with zero-containing
     attention masks (no effect in the reference: the M backbone never reads the attention_bias they are turned into).
The oracle side of every mode is pinned bit-exact to the real reference (tests/test_oracle_golden.py)."""
import contextlib
import io
from types import SimpleNamespace

import pytest
import torch

from helpers import GpuBackedOracleModel, load_golden, tiny_gpu_model
from oracle import generate as G
from oracle import sampling as S

pytestmark = pytest.mark.gpu
MASK = 126336


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def test_generate_image_lockstep_with_oracle():
    from mmada_parallel_b200.generators.image_generation_generator import generate_image
    t = load_golden("trajectory_t2i_tiny.pt")
    model, cfg, _ = tiny_gpu_model(t["meta"])
    backed = GpuBackedOracleModel(model)
    lay = t["layout"]
    for run in t["runs"]:
        common = dict(seq_len=lay["seq_len"], newline_every=lay["newline_every"], code_start=lay["code_start"],
                      uncon_ids=lay["uncon_ids"], text_vocab_size=126356, codebook_size=8192, **run["kwargs"])
        tr_o, tr_g = [], []
        vo = G.generate_image(backed, lay["prompt"], generator=torch.Generator().manual_seed(run["seed"]), trace=tr_o, **common)
        before = lay["prompt"].clone()
        with quiet():
            vg = generate_image(model, lay["prompt"], generator=torch.Generator().manual_seed(run["seed"]), _trace=tr_g, debug=False, **common)
        assert torch.equal(before, lay["prompt"]), "the caller's prompt must not be modified"
        assert len(tr_o) == len(tr_g), (run["name"], len(tr_o), len(tr_g))
        for so, sg in zip(tr_o, tr_g):
            assert so["keep_n"] == sg["keep_n"], (run["name"], so["step"])
            assert torch.equal(so["sampled"].reshape(-1), sg["sampled"].cpu()), (run["name"], so["step"], "sampled")
            assert torch.equal(so["x"], sg["x"].cpu()), (run["name"], so["step"], "ids")
        assert tuple(vg.shape) == (1, lay["seq_len"]) and vg.dtype == torch.int64
        assert torch.equal(vg.cpu(), vo), run["name"]
        assert int((vg == MASK).sum()) == 0
        # agreement with the REAL reference's ids (computed from CPU logits; near-tied logits may legitimately differ)
        print(f"[golden t2i] {run['name']}: agreement with the reference trajectory {float((vg.cpu() == run['vq_ids']).float().mean()):.3f}")
        # the reference's token cache flag is output-invariant (pinned in oracle/make_golden_t2i.py) - here too
        with quiet():
            vc = generate_image(model, lay["prompt"], generator=torch.Generator().manual_seed(run["seed"]), use_cache=True, debug=False, **common)
        assert torch.equal(vc, vg)
    with pytest.raises(AssertionError), quiet():
        generate_image(model, torch.cat([lay["prompt"], lay["prompt"]]), seq_len=16, code_start=lay["code_start"], debug=False)


def _m_model(meta, max_batch=4):
    from mmada_parallel_b200.mmada import MMadaModelLM
    return tiny_gpu_model(meta, cls=MMadaModelLM, max_batch=max_batch)


class _Tok:
    bos_token_id = 126080

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


def test_t2i_generate_m_lockstep_with_oracle():
    t = load_golden("trajectory_m_modes_tiny.pt")
    tv = t["meta"]["text_vocab_len"]
    model, cfg, _ = _m_model(t["meta"])
    backed = GpuBackedOracleModel(model)
    up = SimpleNamespace(text_tokenizer=_Tok(tv))
    for r in t["t2i"]:
        ids_o = r["input_ids"].clone()
        tr = []
        so = G.t2i_generate(backed, ids_o, r["uncond_input_ids"].clone(), attention_mask=r["attention_mask"],
                            uncond_attention_mask=r["attention_mask"], generator=torch.Generator().manual_seed(r["seed"]),
                            text_vocab_len=tv, trace=tr, **r["kwargs"])
        ids_g = r["input_ids"].clone()
        sg = model.t2i_generate(input_ids=ids_g, uncond_input_ids=r["uncond_input_ids"].clone(), attention_mask=r["attention_mask"],
                                uncond_attention_mask=r["attention_mask"], generator=torch.Generator().manual_seed(r["seed"]),
                                uni_prompting=up, **r["kwargs"])
        assert sg.dtype == torch.int64 and tuple(sg.shape) == tuple(so.shape)
        assert torch.equal(sg.cpu(), so), r["name"]
        assert torch.equal(ids_g, ids_o), (r["name"], "input_ids must be updated in place exactly like the reference's")
        print(f"[golden M t2i] {r['name']}: agreement with the reference's sampled ids {float((sg.cpu() == r['sampled']).float().mean()):.3f}")


def _noise64(seed):
    def fn(step, shape):
        return torch.rand(shape, dtype=torch.float64, generator=torch.Generator().manual_seed(seed * 1000 + step))
    return fn


def test_m_text_gumbel_and_padding_masks_lockstep():
    t = load_golden("trajectory_m_modes_tiny.pt")
    tv = t["meta"]["text_vocab_len"]
    model, cfg, _ = _m_model(t["meta"])
    backed = GpuBackedOracleModel(model)
    up = SimpleNamespace(text_tokenizer=_Tok(tv))
    # interleave_generate with text_temperature > 0: the fp64 uniform noise is injected on both sides
    r = t["interleave"][0]
    conf = SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=16, codebook_size=8192)),
                           dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=12)))
    io_, to_ = G.interleave_generate(backed, r["input_ids"], r["uncond_input_ids"], soi_id=126085, eoi_id=126086, bos_id=126080,
                                     mask_id=MASK, num_vq_tokens=16, codebook_size=8192, max_seq_length=12, text_vocab_len=tv,
                                     generator=torch.Generator().manual_seed(r["seed"]), text_noise=_noise64(7), **r["kwargs"])
    ig, tg = model.interleave_generate(input_ids=r["input_ids"], uncond_input_ids=r["uncond_input_ids"],
                                       reserved_token_mapping={"<|soi|>": 126085, "<|eoi|>": 126086},
                                       generator=torch.Generator().manual_seed(r["seed"]), config=conf, uni_prompting=up,
                                       _text_noise=_noise64(7), **r["kwargs"])
    assert torch.equal(ig.cpu(), io_) and torch.equal(tg.cpu(), to_)
    # without injection the product draws from the global RNG of the device like the reference: runs, and is reproducible
    torch.manual_seed(3)
    a = model.interleave_generate(input_ids=r["input_ids"], uncond_input_ids=r["uncond_input_ids"],
                                  reserved_token_mapping={"<|soi|>": 126085, "<|eoi|>": 126086},
                                  generator=torch.Generator().manual_seed(1), config=conf, uni_prompting=up, **r["kwargs"])
    torch.manual_seed(3)
    b = model.interleave_generate(input_ids=r["input_ids"], uncond_input_ids=r["uncond_input_ids"],
                                  reserved_token_mapping={"<|soi|>": 126085, "<|eoi|>": 126086},
                                  generator=torch.Generator().manual_seed(1), config=conf, uni_prompting=up, **r["kwargs"])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # mmu_generate: temperature > 0 (noise of the FULL logits shape [B, L, V]) and a zero-containing attention mask
    for r in t["mmu"]:
        kw = dict(r["kwargs"])
        if kw.get("temperature", 0.0) != 0:
            xo = G.mmu_generate(backed, r["idx"], attention_mask=r["attention_mask"], text_noise=_noise64(11), **kw)
            model._mmu_noise = _noise64(11)
            try:
                xg = model.mmu_generate(idx=r["idx"], attention_mask=r["attention_mask"], **kw)
            finally:
                model._mmu_noise = None
        else:
            xo = G.mmu_generate(backed, r["idx"], attention_mask=r["attention_mask"], **kw)
            xg = model.mmu_generate(idx=r["idx"], attention_mask=r["attention_mask"], **kw)
            assert torch.equal(xg, model.mmu_generate(idx=r["idx"], attention_mask=None, **kw)), "padding masks have no effect (reference quirk)"
        assert torch.equal(xg.cpu(), xo), r["name"]
        assert int((xg == MASK).sum()) == 0


def test_text_step_gumbel64_kernel_vs_oracle():
    """mmdp_text_step_gumbel64 against oracle.sampling.text_step(uniform64=...) on identical inputs: ids bit-exact, fp64 confidence
    at 1e-12, with and without the CFG mix."""
    from mmada_parallel_b200 import _lib as L
    g = torch.Generator().manual_seed(21)
    R, V = 24, 16384
    cond = (torch.randn(R, V, generator=g) * 2).to(torch.bfloat16)
    unc = (torch.randn(R, V, generator=g) * 2).to(torch.bfloat16)
    ids = torch.where(torch.rand(R, generator=g) < 0.7, torch.tensor(MASK), torch.randint(0, V, (R,), generator=g))
    u = torch.rand(R, V, dtype=torch.float64, generator=g)
    for use_cfg, temp in ((False, 0.7), (True, 1.3)):
        new_o, x0_o, conf_o = S.text_step(cond, ids, MASK, 5, uncond_logits=unc if use_cfg else None, text_cfg=1.75 if use_cfg else 0.0,
                                          temperature=temp, uniform64=u)
        c, un, ud = cond.cuda().contiguous(), unc.cuda().contiguous(), u.cuda().contiguous()
        idsd = ids.cuda().clone()
        x0 = torch.empty(R, dtype=torch.int64, device="cuda")
        conf = torch.empty(R, dtype=torch.float64, device="cuda")
        L.check(L.lib.mmdp_text_step_gumbel64(L.ptr(c), L.ptr(un) if use_cfg else None, V, R, V, 1.75 if use_cfg else 0.0, L.ptr(ud), V,
                                              float(temp), L.ptr(idsd), MASK, 5, L.ptr(x0), L.ptr(conf), L.stream_ptr()))
        torch.cuda.synchronize()
        masked = ids == MASK
        assert torch.equal(x0.cpu()[masked], x0_o[masked])
        assert torch.allclose(conf.cpu(), conf_o, rtol=1e-12, atol=0)
        assert torch.equal(idsd.cpu(), new_o)
