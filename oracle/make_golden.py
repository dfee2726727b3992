"""Generates tests/golden/*.pt by running the REAL reference (imported read-only from MMDP_REFERENCE_ROOT) on seeded
inputs, and checks the oracle restatement against it while doing so ("pinning the oracle").

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden

Runs only where a reference checkout is available (MMDP_REFERENCE_ROOT). The fixtures are small (ids, noise seeds,
a few hundred logits) and are committed; tests/test_oracle_golden.py re-checks the oracle against them on every run and
tests/test_gpu_*.py check the CUDA path against them on the H100.
"""
from __future__ import annotations

import contextlib
import io
import os
from types import SimpleNamespace

import torch

from . import generate as G
from . import llada
from . import ref_shim
from . import sampling as S

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

TINY = dict(d_model=256, n_heads=2, n_layers=2, mlp_hidden_size=512, vocab_size=134656, max_sequence_length=512)
WEIGHT_SEED = 1234


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def layout_a(prompt_len=8, grid=4, text_len=16, seed=0):
    """Synthetic A-variant sequence with the structure of A/inference.py:129-156 at reduced size."""
    g = torch.Generator().manual_seed(seed)
    BOA, BOI, EOI, EOA, MASK, NL = 126354, 126349, 126350, 126355, 126336, 126084
    prompt = torch.randint(0, 126000, (prompt_len,), generator=g).tolist()
    img_in = torch.randint(126356, 126356 + 8192, (grid * grid,), generator=g).tolist()
    img = [BOI]
    for r in range(grid):
        img += img_in[r * grid:(r + 1) * grid] + [NL]
    img += [EOI]
    con = prompt[:-1] + img + prompt[-1:]
    pred = [BOA, BOI]
    for r in range(grid):
        pred += [MASK] * grid + [NL]
    pred += [EOI] + [MASK] * text_len + [EOA]
    ids = con + pred
    image_start = len(con) + 2
    text_start = len(con) + 2 + grid * (grid + 1) + 1
    text_end = text_start + text_len
    unc_prompt = torch.randint(0, 126000, (3,), generator=g).tolist()
    uncon_text = unc_prompt[:-1] + img + unc_prompt[-1:]
    uncon_image = prompt
    return dict(input_ids=torch.tensor([ids]), text_start=text_start, text_end=text_end, image_start=image_start,
                seq_len=grid * grid, newline_every=grid, uncon_text=torch.tensor([uncon_text]),
                uncon_image=torch.tensor([uncon_image]))


def main():
    assert ref_shim.available(), "reference tree not found"
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    cfg = llada.make_config(**TINY)
    sd = llada.make_weights(cfg, seed=WEIGHT_SEED)
    with quiet():
        ref = ref_shim.build_ref_model_a(cfg, sd)
    _, _, pg, _ = ref_shim.load_a()
    oracle_model = llada.OracleModel(cfg, sd)
    meta = dict(tiny=TINY, weight_seed=WEIGHT_SEED)

    # ---- 1. forward logits ---------------------------------------------------------------------------------
    lay = layout_a()
    ids = lay["input_ids"]
    with torch.no_grad():
        lr = ref(ids, infer=True, use_cache=False).logits
    lo = oracle_model(ids).logits
    assert torch.equal(lr, lo), "oracle forward != reference forward"
    ids2 = torch.cat([ids, ids.flip(1)], dim=0)  # batch of 2 equal-length rows (CFG batch)
    with torch.no_grad():
        lr2 = ref(ids2, infer=True, use_cache=False).logits
    assert torch.equal(lr2, oracle_model(ids2).logits)
    cols = torch.cat([torch.arange(0, 134656, 997), torch.arange(126356, 126356 + 8192, 61)])
    top = lr.float().topk(2, dim=-1)
    torch.save(dict(meta=meta, ids=ids, ids2=ids2, cols=cols, logits_cols=lr[0][:, cols].clone(),
                    logits2_cols=lr2[:, :, cols].clone(), argmax=lr[0].argmax(-1), top2_vals=top.values[0].clone(),
                    top2_idx=top.indices[0].clone()), os.path.join(OUT, "forward_tiny.pt"))
    print("forward_tiny ok", tuple(lr.shape))

    # ---- 2. sampler known-answer tests from the reference functions ------------------------------------------------
    kat = dict(meta=meta)
    # A: mask_by_random_topk / add_gumbel_noise / get_num_transfer_tokens
    cases = []
    for seed, n, k, temp in [(0, 1024, 1, 0.5), (1, 1024, 700, 0.9), (2, 1024, 1023, 0.0), (3, 64, 10, 1.0), (4, 1024, 5000, 0.3)]:
        g0 = torch.Generator().manual_seed(100 + seed)
        probs = torch.softmax(torch.randn(n, generator=g0) * 3, -1).to(torch.bfloat16)[None]
        probs[0, ::7] = torch.finfo(torch.bfloat16).max
        g1 = torch.Generator().manual_seed(seed)
        masking = pg.mask_by_random_topk(torch.tensor([[k]]), probs, temp, generator=g1)
        g2 = torch.Generator().manual_seed(seed)
        noise = torch.randn(probs.shape, dtype=probs.dtype, generator=g2)
        mo, _ = S.mask_by_random_topk_a(k, probs[0], temp, noise[0])
        assert torch.equal(masking[0], mo), f"A mask_by_random_topk mismatch (seed {seed})"
        cases.append(dict(probs=probs[0], k=k, temp=temp, noise=noise[0], masking=masking[0]))
    kat["a_mask_by_random_topk"] = cases
    # probe of this machine's torch.sort(stable=False) tie order (see sampling.mask_by_random_topk_a)
    probe = (torch.randn(1, 1024, generator=torch.Generator().manual_seed(77)) * 2).to(torch.bfloat16)
    kat["sort_probe"] = dict(x=probe, idx=torch.sort(probe, dim=-1, descending=False).indices)
    cases = []
    for seed, temp in [(0, 0.7), (1, 1.3)]:
        logits = (torch.randn(1, 6, 4096, generator=torch.Generator().manual_seed(seed)) * 2).to(torch.bfloat16)
        out = pg.add_gumbel_noise(logits, temp, generator=torch.Generator().manual_seed(seed + 50))
        u = torch.rand(logits.shape, dtype=logits.dtype, generator=torch.Generator().manual_seed(seed + 50))
        assert torch.equal(out, S.add_gumbel_noise_a(logits, temp, u))
        cases.append(dict(logits=logits[0], temp=temp, uniform=u[0], out=out[0], argmax=out[0].argmax(-1)))
    kat["a_add_gumbel_noise"] = cases
    ntt = {}
    for n, steps in [(256, 128), (16, 8), (100, 7), (5, 9), (0, 4)]:
        m = torch.zeros(1, max(n, 1), dtype=torch.bool)
        m[0, :n] = True
        r = pg.get_num_transfer_tokens(m, steps)[0].tolist()
        assert r == S.get_num_transfer_tokens_a(n, steps)
        ntt[(n, steps)] = r
    kat["a_num_transfer"] = ntt
    kat["a_sched_len_1024_128"] = [S.sched_len(1024, s, 128) for s in range(128)]
    ref_sched = [int((1024 * pg.cosine_schedule(torch.tensor(1.0 * (s + 1) / 128))).floor().item()) for s in range(128)]
    assert ref_sched == kat["a_sched_len_1024_128"] and ref_sched[-1] == -1
    assert S.image_step_indices(128, 64) == torch.linspace(128 // 4, 127, 64).round().int().tolist()
    # M
    mm, sm, mv = ref_shim.load_m()
    cases = []
    for seed, n, k, temp in [(0, 1024, 1, 0.5), (1, 1024, 300, 0.9), (2, 1024, 1022, 0.0), (3, 64, 10, 1.0)]:
        g0 = torch.Generator().manual_seed(200 + seed)
        probs = torch.softmax(torch.randn(n, generator=g0) * 3, -1).to(torch.bfloat16)[None]
        probs[0, ::5] = torch.finfo(torch.bfloat16).max
        masking = sm.mask_by_random_topk(torch.tensor([[k]]), probs, temp, generator=torch.Generator().manual_seed(seed))
        u = torch.zeros_like(probs).uniform_(0, 1, generator=torch.Generator().manual_seed(seed))
        mo, _ = S.mask_by_random_topk_m(k, probs[0], temp, u[0])
        assert torch.equal(masking[0], mo), f"M mask_by_random_topk mismatch (seed {seed})"
        cases.append(dict(probs=probs[0], k=k, temp=temp, noise=u[0], masking=masking[0]))
    kat["m_mask_by_random_topk"] = cases
    ntt = {}
    for n, steps in [(255, 128), (16, 8), (100, 7), (5, 9)]:
        m = torch.zeros(1, n, dtype=torch.bool)
        m[0, :n] = True
        r = mm.get_num_transfer_tokens(m, steps)[0].tolist()
        assert r == S.get_num_transfer_tokens_m(n, steps)
        ntt[(n, steps)] = r
    kat["m_num_transfer"] = ntt
    if mv is not None:
        with quiet():
            lfq = mv.LFQuantizer(codebook_dim=13)
        idx = torch.randint(0, 8192, (2, 64), generator=torch.Generator().manual_seed(5))
        zq = lfq.get_codebook_entry(idx)  # [B, 13, 8, 8]
        assert torch.equal(zq.reshape(2, 13, 64), S.lfq_codebook_entry(idx, 13))
        kat["m_lfq"] = dict(idx=idx, zq=zq.reshape(2, 13, 64))
    torch.save(kat, os.path.join(OUT, "sampler_kat.pt"))
    print("sampler_kat ok")

    # ---- 3. full trajectories, variant A -------------------------------------------------------------------
    traj = dict(meta=meta, layout=lay, runs=[])
    for name, kw, seed in [
        ("greedy_cfgimg4", dict(temperature=0.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0), 42),
        ("canonical_temp1", dict(temperature=1.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0), 42),
        ("both_cfg_texttemp", dict(temperature=1.0, text_temperature=0.7, cfg_scale=1.5, cfg_img=4.0), 7),
        ("no_cfg", dict(temperature=1.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=0.0), 3),
    ]:
        common = dict(text_steps=8, text_gen_length=16, text_block_length=4, timesteps=4, tokenizer=None,
                      text_vocab_size=126356, codebook_size=8192, **kw)
        args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
        torch.manual_seed(999)
        with quiet():
            img_r, txt_r = pg.generate_ti2ti(ref, lay["input_ids"], generator=torch.Generator().manual_seed(seed), **args, **common)
        torch.manual_seed(999)
        trace = []
        img_o, txt_o = G.generate_ti2ti(oracle_model, lay["input_ids"], generator=torch.Generator().manual_seed(seed),
                                        trace=trace, **args, **common)
        assert img_r == img_o and txt_r == txt_o, f"A trajectory {name}: oracle != reference"
        traj["runs"].append(dict(name=name, kwargs=common, seed=seed, global_seed=999, image_tokens=img_r, text_tokens=txt_r,
                                 trace=[{k: v for k, v in t.items()} for t in trace]))
        print("trajectory A", name, "ok; masked text left:", 16 - len(txt_r))
    torch.save(traj, os.path.join(OUT, "trajectory_a_tiny.pt"))

    # ---- 4. full trajectory, variant M ---------------------------------------------------------------------
    mcfg = mm.MMadaConfig(**{k: v for k, v in ref_shim.ref_config_a(cfg).to_dict().items()
                             if k not in ("architectures", "model_type", "transformers_version", "mask_token_id")}, mask_token_id=126336)
    mcfg.use_cache = False
    with quiet():
        refm = mm.MMadaModelLM(mcfg, init_params=False).eval().to(torch.bfloat16)
    missing, unexpected = refm.load_state_dict(sd, strict=False)
    assert not unexpected
    g = torch.Generator().manual_seed(11)
    NVQ, MAXSEQ, TVOC = 16, 12, 126349
    soi, eoi, bos = 126084 + 1, 126084 + 2, 126080
    inp = torch.cat([torch.tensor([126340, soi]), torch.randint(TVOC, TVOC + 8192, (NVQ,), generator=g), torch.tensor([eoi]),
                     torch.randint(0, 126000, (6,), generator=g)])
    unc = inp.clone()
    unc[-6:] = torch.randint(0, 126000, (6,), generator=g)
    conf = SimpleNamespace(model=SimpleNamespace(mmada=SimpleNamespace(num_vq_tokens=NVQ, codebook_size=8192)),
                           dataset=SimpleNamespace(preprocessing=SimpleNamespace(max_seq_length=MAXSEQ)))

    class Tok:
        bos_token_id = bos

        def __len__(self):
            return TVOC

    up = SimpleNamespace(text_tokenizer=Tok())
    mruns = []
    for name, kw, seed in [("m_canonical", dict(text_cfg=2.5, image_cfg=4.0, text_steps=8, image_steps=4), 42),
                           ("m_imgcfg_only", dict(text_cfg=0.0, image_cfg=3.5, text_steps=6, image_steps=6), 5)]:
        with quiet():
            img_r, txt_r = refm.interleave_generate(input_ids=inp, uncond_input_ids=unc, reserved_token_mapping={"<|soi|>": soi, "<|eoi|>": eoi},
                                                    generator=torch.Generator().manual_seed(seed), config=conf, uni_prompting=up, **kw)
        trace = []
        img_o, txt_o = G.interleave_generate(oracle_model, inp, unc, soi_id=soi, eoi_id=eoi, bos_id=bos, mask_id=126336,
                                             num_vq_tokens=NVQ, codebook_size=8192, max_seq_length=MAXSEQ, text_vocab_len=TVOC,
                                             generator=torch.Generator().manual_seed(seed), trace=trace, **kw)
        assert torch.equal(img_r, img_o) and torch.equal(txt_r, txt_o), f"M trajectory {name}: oracle != reference"
        mruns.append(dict(name=name, kwargs=kw, seed=seed, image_ids=img_r, text_ids=txt_r, trace=trace))
        print("trajectory M", name, "ok")
    torch.save(dict(meta=meta, input_ids=inp, uncond_input_ids=unc, soi=soi, eoi=eoi, bos=bos, mask_id=126336, num_vq_tokens=NVQ,
                    max_seq_length=MAXSEQ, text_vocab_len=TVOC, runs=mruns), os.path.join(OUT, "trajectory_m_tiny.pt"))
    print("all golden fixtures written to", OUT)


if __name__ == "__main__":
    main()
