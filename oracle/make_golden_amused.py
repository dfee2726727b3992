"""Writes the aMUSEd VQ-VAE fixtures (variant A's tokenizer). Needs MMDP_REFERENCE_ROOT for the glue and trajectory parts.

    PYTHONDONTWRITEBYTECODE=1 MMDP_REFERENCE_ROOT=... python -m oracle.make_golden_amused

  tests/golden/amused_vq.pt          oracle/amused.py decode / encode / quantize outputs ("small" configs with and without
                                     mid-block attention; the "full" aMUSEd 512 config at 32x32 and 64x16 latent grids). The
                                     oracle is restated from diffusers' structure and NOT pinned against diffusers (see its
                                     docstring): these fixtures pin the native VQModel to the oracle only.
  tests/golden/amused_glue.pt        the REAL MMaDA-Parallel-A/utils/image_utils.py, imported with `diffusers` stubbed by the
                                     oracle (VQModel -> amused.OracleVQModel, VaeImageProcessor -> amused.VaeImageProcessor):
                                     decode_vq_to_image images, encode_img_with_breaks / encode_img_with_paint ids and
                                     visualisations, and the crop helpers under seeded `random`.
  tests/golden/trajectory_paint_tiny.pt   the REAL generate_ti2ti on the tiny model of make_golden.py with inpainting and
                                     outpainting inputs built as A/inference.py:120-158 builds them (checked against the oracle loop).
"""
from __future__ import annotations

import contextlib
import hashlib
import importlib
import io
import os
import random
import sys
import types

import numpy as np
import torch
from PIL import Image

from . import amused as AM
from . import generate as G
from . import llada, ref_shim
from .make_golden import TINY, WEIGHT_SEED

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

SMALL = dict(block_out_channels=(32, 64), layers_per_block=1, latent_channels=16, num_vq_embeddings=512)
# five levels (16 pixels per token, like aMUSEd) at small widths: the glue fixtures and the paint trajectory
GLUE = dict(block_out_channels=(32, 32, 32, 32, 64), layers_per_block=1, latent_channels=16, num_vq_embeddings=512,
            mid_block_add_attention=True)


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def pixels(seed, b, h, w):
    return torch.rand(b, 3, h, w, generator=torch.Generator().manual_seed(seed))


def test_image(seed, w, h):
    """Smooth colour ramps plus seeded noise: a picture with structure at several scales."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 100 * np.sin(xx / (7 + seed)), 128 + 100 * np.cos(yy / 11), (xx + yy) * 255 / (w + h)], -1)
    arr = np.clip(base + g.normal(0, 20, base.shape), 0, 255).astype(np.uint8)
    return Image.fromarray(arr)


def digest(img) -> tuple:
    """(shape, sha256) of an image's uint8 pixels: exact comparison without storing the pixels."""
    a = np.ascontiguousarray(np.asarray(img))
    return tuple(a.shape), hashlib.sha256(a.tobytes()).hexdigest()


def vq_fixtures():
    out = {}
    for tag, kw, seed, cases in (
        ("small_attn", dict(SMALL, mid_block_add_attention=True), 21, [(2, 8, 8), (1, 6, 10)]),
        ("small_noattn", dict(SMALL, mid_block_add_attention=False), 22, [(2, 8, 8), (1, 12, 4)]),
        ("full", dict(mid_block_add_attention=False), 23, [(1, 32, 32), (1, 64, 16)]),
    ):
        cfg = AM.make_config(**kw)
        w = AM.make_weights(cfg, seed)
        scale = 2 ** (len(cfg.block_out_channels) - 1)
        stride = 1 if tag != "full" else 8
        lat_stride = 1 if tag != "full" else 2  # full config: latents / ids of every other latent row (fixture size)
        runs = []
        for ci, (b, h, wd) in enumerate(cases):
            ids = torch.randint(0, cfg.num_vq_embeddings, (b, h, wd), generator=torch.Generator().manual_seed(seed * 10 + ci))
            img = AM.decode(ids, w, cfg, force_not_quantize=True, shape=(b, h, wd, cfg.latent_channels))
            px_seed = seed * 10 + ci + 500
            lat = AM.encode(pixels(px_seed, b, h * scale, wd * scale), w, cfg)
            _, qidx = AM.quantize(lat, w)
            runs.append(dict(batch=b, h=h, w=wd, ids=ids, stride=stride, image=img[:, :, ::stride, ::stride].clone(),
                             mean=float(img.mean()), std=float(img.std()), shape=tuple(img.shape), pixel_seed=px_seed,
                             lat_stride=lat_stride, latents=lat[:, :, ::lat_stride].clone(),
                             quant_ids=qidx.view(b, h, wd)[:, ::lat_stride].reshape(-1).clone()))
            print(tag, (b, h, wd), "image std", round(float(img.std()), 3), "latent std", round(float(lat.std()), 3))
        out[tag] = dict(cfg=kw, weight_seed=seed, runs=runs)
    torch.save(out, os.path.join(OUT, "amused_vq.pt"))


def load_ref_image_utils():
    """The reference module with `diffusers` replaced by the oracle's restatement."""
    d = types.ModuleType("diffusers")
    d.VQModel = AM.OracleVQModel
    dp = types.ModuleType("diffusers.image_processor")
    dp.VaeImageProcessor = AM.VaeImageProcessor
    sys.modules["diffusers"] = d
    sys.modules["diffusers.image_processor"] = dp
    if ref_shim.REF_A not in sys.path:
        sys.path.insert(0, ref_shim.REF_A)
    sys.modules.pop("utils.image_utils", None)
    return importlib.import_module("utils.image_utils")


def glue_fixtures(iu, vq):
    out = dict(cfg=GLUE, weight_seed=31)
    # decode_vq_to_image
    dec = []
    for i, (hh, ww) in enumerate(((128, 128), (96, 256))):
        n = (hh // 16) * (ww // 16)
        ids = torch.randint(0, GLUE["num_vq_embeddings"], (1, n), generator=torch.Generator().manual_seed(40 + i))
        img = iu.decode_vq_to_image(ids, None, None, hh, ww, vq)
        dec.append(dict(ids=ids, height=hh, width=ww, image=np.asarray(img).copy()))
    out["decode"] = dec
    # encode_img_with_breaks and encode_img_with_paint
    image_args = ((1, 256, 256), (2, 384, 192), (3, 250, 200))
    images = [test_image(*a) for a in image_args]
    # regenerated by the tests with test_image(); the digests check that the regeneration is the same picture
    out["image_sources"] = [dict(args=a, digest=digest(im)) for a, im in zip(image_args, images)]
    out["breaks"] = [iu.encode_img_with_breaks(im, vq) for im in images]
    out["indices"] = []
    for im in images:
        x = AM.preprocess(im, 16)
        lat = vq.encode(x).latents
        out["indices"].append(dict(ids=vq.quantize(lat)[2][2].clone(), lat_h=lat.shape[2], lat_w=lat.shape[3],
                                   Hp=x.shape[2], Wp=x.shape[3]))
    paint = []
    for ii in range(len(images)):
        for mode in ("inpainting", "outpainting"):
            for hr, wr in ((1.0, 0.2), (0.5, 0.5), (0.37, 0.81)):
                for ds in ("area", "nearest", "bilinear"):
                    for dil in (0, 1):
                        kw = dict(mask_h_ratio=hr, mask_w_ratio=wr, gray_value=127, downsample_mode=ds, dilate_latent_k=dil,
                                  mask_mode=mode)
                        tokens, vis = iu.encode_img_with_paint(images[ii], vq, **kw)
                        paint.append(dict(image=ii, kwargs=kw, tokens=torch.tensor(tokens, dtype=torch.int32), vis=digest(vis)))
    out["paint"] = paint
    # layout and crop helpers
    out["crop_lists"] = {(n, p, r): iu.generate_crop_size_list(n, p, r) for n, p, r in ((256, 32, 4.0), (64, 16, 2.0), (100, 8, 4.0))}
    crops = []
    src = [test_image(4, 640, 480), test_image(5, 300, 1000), test_image(6, 1200, 1200)]
    for si, im in enumerate(src):
        for seed in (0, 1):
            random.seed(seed)
            a = iu.var_center_crop(im, crop_size_list=iu.generate_crop_size_list((512 // 32) ** 2, 32))
            random.seed(seed)
            b = iu.center_crop(im, (256, 128))
            crops.append(dict(src=si, seed=seed, var=digest(a), center=digest(b)))
    out["crop_sources"] = [dict(args=a, digest=digest(im)) for a, im in zip(((4, 640, 480), (5, 300, 1000), (6, 1200, 1200)), src)]
    out["crops"] = crops
    out["break_lines"] = [(list(range(12)), 3, 4, 9, iu.add_break_line(list(range(12)), 3, 4, 9)),
                          (list(range(6)), 2, 3, 0, iu.add_break_line(list(range(6)), 2, 3))]
    out["vq_params"] = {(h, w, s): iu.calculate_vq_params(h, w, s) for h, w, s in ((512, 512, 16), (256, 1024, 16), (384, 640, 8))}
    torch.save(out, os.path.join(OUT, "amused_glue.pt"))
    print("amused_glue ok:", len(paint), "paint cases")


def paint_trajectory(iu, vq):
    cfg = llada.make_config(**TINY)
    sd = llada.make_weights(cfg, seed=WEIGHT_SEED)
    with quiet():
        ref = ref_shim.build_ref_model_a(cfg, sd)
    _, _, pg, _ = ref_shim.load_a()
    oracle_model = llada.OracleModel(cfg, sd)
    BOA, BOI, EOI, EOA, MASK, NL = 126354, 126349, 126350, 126355, 126336, 126084
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, 126000, (8,), generator=g).tolist()
    unc_prompt = torch.randint(0, 126000, (3,), generator=g).tolist()
    img = test_image(7, 64, 64)                                   # 4 x 4 tokens at 16 pixels per token
    input_img_token = iu.encode_img_with_breaks(img, vq)
    con = prompt[:-1] + input_img_token + prompt[-1:]
    uncon_text = unc_prompt[:-1] + input_img_token + unc_prompt[-1:]
    text_len = 16
    runs = []
    for mode, hr, wr in (("inpainting", 0.5, 0.5), ("outpainting", 1.0, 0.5)):
        img_mask_token, _ = iu.encode_img_with_paint(img, vqvae=vq, mask_h_ratio=hr, mask_w_ratio=wr, mask_mode=mode)
        pred = [BOA, BOI] + img_mask_token + [EOI] + [MASK] * text_len + [EOA]
        image_start = len(con) + 2
        text_start = image_start + len(img_mask_token) + 1
        lay = dict(input_ids=torch.tensor([con + pred]), text_start=text_start, text_end=text_start + text_len,
                   image_start=image_start, seq_len=16, newline_every=4, uncon_text=torch.tensor([uncon_text]),
                   uncon_image=torch.tensor([prompt]))
        for name, kw, seed in (("greedy", dict(temperature=0.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0), 42),
                               ("temp1", dict(temperature=1.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0), 42)):
            common = dict(text_steps=8, text_gen_length=text_len, text_block_length=4, timesteps=4, tokenizer=None,
                          text_vocab_size=126356, codebook_size=8192, **kw)
            args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
            torch.manual_seed(999)
            with quiet():
                img_r, txt_r = pg.generate_ti2ti(ref, lay["input_ids"], generator=torch.Generator().manual_seed(seed), **args, **common)
            torch.manual_seed(999)
            trace = []
            img_o, txt_o = G.generate_ti2ti(oracle_model, lay["input_ids"], generator=torch.Generator().manual_seed(seed), trace=trace,
                                            **args, **common)
            assert img_r == img_o and txt_r == txt_o, f"paint trajectory {mode}/{name}: oracle != reference"
            runs.append(dict(name=f"{mode}_{name}", mode=mode, layout=lay, kwargs=common, seed=seed, global_seed=999,
                             image_tokens=img_r, text_tokens=txt_r, trace=trace))
            print("paint trajectory", mode, name, "ok; masked image cells:", img_mask_token.count(MASK))
    torch.save(dict(meta=dict(tiny=TINY, weight_seed=WEIGHT_SEED), runs=runs), os.path.join(OUT, "trajectory_paint_tiny.pt"))


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    os.makedirs(OUT, exist_ok=True)
    vq_fixtures()
    assert ref_shim.available(), "reference tree not found (MMDP_REFERENCE_ROOT)"
    iu = load_ref_image_utils()
    gcfg = AM.make_config(**GLUE)
    vq = AM.OracleVQModel(gcfg, AM.make_weights(gcfg, 31))
    glue_fixtures(iu, vq)
    paint_trajectory(iu, vq)


if __name__ == "__main__":
    main()
