"""A "well-separated" tiny model on which the greedy AND the stochastic generate_ti2ti trajectories are decided with margins far
above the floating-point tolerance of a GPU forward, so that a correct implementation must reproduce the REAL reference's
token ids bit for bit on every step (VERDICT r01 weak #3: the random-weight fixtures only allow agreement "where the margin
allows"). Writes tests/golden/trajectory_a_separated.pt.

    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_separated

Construction: the tiny LLaDA of the other fixtures, but the LM head keeps only a few LIVE rows (24 text tokens, 16 VQ codes,
gain 4); every other row is scaled by 1e-3, so logits have a handful of well-spread candidates instead of 134 656 near-ties.
A seed is accepted when the oracle trajectory is unchanged under N_PERTURB independent perturbations of the logits by +-3 bf16
ulp of the logit scale (the GPU test first checks that its logits are inside this radius of the oracle's; dead rows are perturbed in proportion to their row
norm, as accumulation error is) - every decision (argmax, top-k confidence rank, sampling race, re-mask cut) then has more than
that margin with overwhelming probability. The accepted configuration is run through the REAL reference, which must agree
with the unperturbed oracle, and its per-step ids are stored.
"""
from __future__ import annotations

import os
from types import SimpleNamespace

import torch

from . import generate as G
from . import llada
from . import ref_shim
from .make_golden import OUT, TINY, layout_a, quiet

N_LIVE_TEXT, N_LIVE_VQ, GAIN, DEAD = 24, 16, 4.0, 1e-3
RUNS = [("greedy", dict(text_steps=4, timesteps=2, text_gen_length=8, temperature=0.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0)),
        ("bench_like", dict(text_steps=4, timesteps=2, text_gen_length=8, temperature=1.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0)),
        ("both_cfg_gumbel", dict(text_steps=4, timesteps=2, text_gen_length=8, temperature=0.8, text_temperature=0.5, cfg_scale=1.5, cfg_img=3.0))]
# 32 perturbations: with 8, a seed was accepted whose bench-like trajectory an H100 forward inside the radius still flipped
N_PERTURB = 32
PERTURB_ULPS = 3.0   # measured GPU error on these models: up to 2.5 bf16 ulp of the logit scale (a single bf16 rounding step of the largest logits is already 1.6); the test re-checks <= 3


def separated_weights(cfg, seed: int):
    """Deterministic recipe (re-materialised by the tests from the seed): make_weights + live/dead head rows."""
    sd = llada.make_weights(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 999)
    live_t = torch.randperm(126000, generator=g)[:N_LIVE_TEXT]
    live_v = 126356 + torch.randperm(8192, generator=g)[:N_LIVE_VQ]
    head = sd["model.transformer.ff_out.weight"].float()
    scale = torch.full((head.shape[0], 1), DEAD)
    scale[live_t] = GAIN
    scale[live_v] = GAIN
    sd["model.transformer.ff_out.weight"] = (head * scale).to(torch.bfloat16)
    return sd, scale[:, 0]


class PerturbedModel:
    """Oracle model whose logits are perturbed like an implementation within `ulps` bf16 ulp of the logit scale."""

    def __init__(self, base, row_gain, ulps: float, seed: int):
        self.base, self.g, self.ulps = base, row_gain / row_gain.max(), ulps
        self.gen = torch.Generator().manual_seed(seed)
        self.device = torch.device("cpu")

    def __call__(self, ids, infer=True, use_cache=False, **_):
        lg = self.base(ids).logits.float()
        scale = lg.abs().max()
        amp = self.ulps * 2.0 ** -8 * torch.maximum(lg.abs(), self.g.to(lg.dtype) * scale)
        noise = (torch.rand(lg.shape, generator=self.gen) * 2 - 1) * amp
        return SimpleNamespace(logits=(lg + noise).to(torch.bfloat16))


def trajectory(model, lay, kw, seed, global_seed):
    torch.manual_seed(global_seed)
    tr = []
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    img, txt = G.generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(seed), trace=tr, stable_sort=True, **args, **kw)
    return img, txt, tr


def main():
    assert ref_shim.available(), "reference tree not found"
    torch.set_num_threads(8)
    cfg = llada.make_config(**TINY)
    lay = layout_a(prompt_len=6, grid=3, text_len=8, seed=5)
    out = dict(meta=dict(tiny=TINY, n_live_text=N_LIVE_TEXT, n_live_vq=N_LIVE_VQ, gain=GAIN, dead=DEAD, layout_seed=5, perturb_ulps=PERTURB_ULPS, layout=dict(prompt_len=6, grid=3, text_len=8)), runs=[])
    for name, kw in RUNS:
        found = None
        for wseed in range(4000, 6000):
            sd, gain = separated_weights(cfg, wseed)
            om = llada.OracleModel(cfg, sd)
            img, txt, tr = trajectory(om, lay, kw, seed=wseed + 1, global_seed=wseed + 2)
            ok = True
            for p in range(N_PERTURB):
                i2, t2, _ = trajectory(PerturbedModel(om, gain, PERTURB_ULPS, 100 * wseed + p), lay, kw, seed=wseed + 1, global_seed=wseed + 2)
                if i2 != img or t2 != txt:
                    ok = False
                    break
            print(f"{name}: weight seed {wseed} {'accepted' if ok else 'rejected (a perturbed run diverged)'}", flush=True)
            if ok:
                found = (wseed, sd, img, txt, tr)
                break
        assert found is not None, name
        wseed, sd, img, txt, tr = found
        with quiet():
            ref = ref_shim.build_ref_model_a(cfg, sd)
        _, _, pg, _ = ref_shim.load_a()
        args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
        torch.manual_seed(wseed + 2)
        with quiet():
            ri, rt = pg.generate_ti2ti(ref, lay["input_ids"], generator=torch.Generator().manual_seed(wseed + 1), **args, **kw)
        assert ri == img and rt == txt, f"{name}: oracle != REAL reference on the separated model"
        out["runs"].append(dict(name=name, kwargs=kw, weight_seed=wseed, seed=wseed + 1, global_seed=wseed + 2, image_tokens=ri, text_tokens=rt,
                                ids_after_text=[r["ids_after_text"] for r in tr],
                                ids_after_image={r["step"]: r["ids_after_image"] for r in tr if "ids_after_image" in r}))
        print(f"{name}: pinned to the real reference ({len(rt)} text tokens, {len(ri)} image tokens)")
    out["layout"] = lay
    torch.save(out, os.path.join(OUT, "trajectory_a_separated.pt"))


if __name__ == "__main__":
    main()
