"""The aMUSEd VQ-VAE oracle (oracle/amused.py) and the product's variant-A host glue, without a GPU.

The oracle is restated from diffusers' structure, not pinned against diffusers (see its docstring); these tests check its
internal properties. The glue checks are exact: tests/golden/amused_glue.pt was recorded from the REAL
A/utils/image_utils.py run over the oracle, and every host-side step of the product (crop sizes, crops, break lines, paint
masks, token layout, visualisation) must reproduce it given the fixture's VQ ids."""
import hashlib
import random

import numpy as np
import pytest
import torch

from helpers import load_golden
from oracle import amused as AM


def _digest(img):
    a = np.ascontiguousarray(np.asarray(img))
    return tuple(a.shape), hashlib.sha256(a.tobytes()).hexdigest()


def glue_images(g):
    """The glue fixture's input pictures, regenerated from their seeds and checked against the recorded digests."""
    from oracle.make_golden_amused import test_image
    out = []
    for s in g["image_sources"]:
        im = test_image(*s["args"])
        assert _digest(im) == tuple(s["digest"])
        out.append(im)
    return out


def _small(attn=True):
    return AM.make_config(block_out_channels=(32, 64), layers_per_block=1, latent_channels=16, num_vq_embeddings=512,
                          mid_block_add_attention=attn)


def test_param_shapes_and_forward_shapes():
    for attn in (True, False):
        cfg = _small(attn)
        sh = AM.param_shapes(cfg)
        w = AM.make_weights(cfg, 0)
        assert set(w) == set(sh) and all(tuple(w[k].shape) == sh[k] for k in sh)
        assert ("encoder.mid_block.attentions.0.to_q.weight" in sh) == attn
        # up_blocks run in reversed channel order: 64 -> 64, then 64 -> 32
        assert "decoder.up_blocks.0.resnets.0.conv_shortcut.weight" not in sh
        assert sh["decoder.up_blocks.1.resnets.0.conv_shortcut.weight"] == (32, 64, 1, 1)
        assert "decoder.up_blocks.1.upsamplers.0.conv.weight" not in sh and "encoder.down_blocks.1.downsamplers.0.conv.weight" not in sh
        assert sh["quantize.embedding.weight"] == (512, 16)
        x = torch.rand(2, 3, 12, 20)
        lat = AM.encode(x, w, cfg)
        assert lat.shape == (2, 16, 6, 10)
        zq, idx = AM.quantize(lat, w)
        assert zq.shape == lat.shape and idx.shape == (120,) and idx.dtype == torch.int64
        assert AM.decode(lat, w, cfg).shape == (2, 3, 12, 20)
        assert AM.decode(lat, w, cfg, force_not_quantize=True, lookup_from_codebook=False).shape == (2, 3, 12, 20)
    full = AM.make_config()
    sh = AM.param_shapes(full)
    assert sh["decoder.conv_in.weight"] == (768, 64, 3, 3) and sh["decoder.conv_out.weight"] == (3, 128, 3, 3)
    assert sum(k.startswith("decoder.up_blocks.0.resnets.") and k.endswith("conv1.weight") for k in sh) == 3


def test_get_codebook_entry_ordering():
    cfg = _small()
    w = AM.make_weights(cfg, 1)
    ids = torch.randint(0, 512, (2, 3, 5), generator=torch.Generator().manual_seed(0))
    z = AM.get_codebook_entry(ids, w, (2, 3, 5, 16))
    emb = w["quantize.embedding.weight"]
    for b in range(2):
        for y in range(3):
            for x in range(5):
                assert torch.equal(z[b, :, y, x], emb[ids[b, y, x]])
    # quantize's flat indices are in (b, y, x) order: decoding them with that shape gives z_q back
    zq, idx = AM.quantize(z + 1e-3, w)
    assert torch.equal(idx.view(2, 3, 5), ids)
    assert torch.allclose(zq, z, atol=1e-6)


def gap_tolerance(z, emb):
    """1e-5 (|z|^2 + max_k |e_k|^2) per latent vector: the fp64 margin beyond which fp32 evaluation cannot swap winners."""
    return 1e-5 * ((z.double() ** 2).sum(1) + (emb.double() ** 2).sum(1).max())


def test_quantize_matches_fp64_argmin_where_decided():
    g = load_golden("amused_vq.pt")
    n_checked = 0
    for tag in ("small_attn", "small_noattn"):
        cfg = AM.make_config(**g[tag]["cfg"])
        w = AM.make_weights(cfg, g[tag]["weight_seed"])
        emb = w["quantize.embedding.weight"]
        for run in g[tag]["runs"]:
            lat = run["latents"]
            z = lat.permute(0, 2, 3, 1).reshape(-1, lat.shape[1])
            d = torch.cdist(z.double(), emb.double()) ** 2
            top2 = d.topk(2, largest=False)
            decided = (top2.values[:, 1] - top2.values[:, 0]) > gap_tolerance(z, emb)
            _, idx = AM.quantize(lat, w)
            assert torch.equal(idx[decided], top2.indices[decided, 0])
            assert torch.equal(idx, run["quant_ids"])
            n_checked += int(decided.sum())
    assert n_checked > 200


def test_oracle_reproduces_small_fixtures():
    g = load_golden("amused_vq.pt")
    for tag in ("small_attn", "small_noattn"):
        cfg = AM.make_config(**g[tag]["cfg"])
        w = AM.make_weights(cfg, g[tag]["weight_seed"])
        for run in g[tag]["runs"]:
            img = AM.decode(run["ids"], w, cfg, force_not_quantize=True, shape=(run["batch"], run["h"], run["w"], cfg.latent_channels))
            assert torch.allclose(img, run["image"], atol=1e-5)


def test_vqmodel_config_validation():
    from mmada_parallel_b200.vqmodel import VQModel
    base = dict(AM.AMUSED_CONFIG, down_block_types=("DownEncoderBlock2D",) * 5, up_block_types=("UpDecoderBlock2D",) * 5)
    for bad in (dict(norm_type="spatial"), dict(act_fn="gelu"), dict(norm_num_groups=16), dict(remap="x.npy"),
                dict(down_block_types=("AttnDownEncoderBlock2D",) * 5), dict(up_block_types=("UpDecoderBlock2D",) * 4),
                dict(block_out_channels=(128, 256, 256, 512, 760)), dict(latent_channels=300), dict(vq_embed_dim=32)):
        with pytest.raises(ValueError):
            VQModel(**dict(base, **bad))


# ---- host glue against the reference's own glue ------------------------------------------------------------------
def test_layout_helpers_match_reference():
    from mmada_parallel_b200.utils import image_utils as IU
    g = load_golden("amused_glue.pt")
    for (n, p, r), want in g["crop_lists"].items():
        assert IU.generate_crop_size_list(n, p, r) == want
    for seq, H, W, nl, want in g["break_lines"]:
        assert IU.add_break_line(seq, H, W, nl) == want
    for (h, w, s), want in g["vq_params"].items():
        assert tuple(IU.calculate_vq_params(h, w, s)) == tuple(want)


def test_crops_match_reference():
    from mmada_parallel_b200.utils import image_utils as IU
    from oracle.make_golden_amused import test_image
    g = load_golden("amused_glue.pt")
    src = []
    for s in g["crop_sources"]:
        im = test_image(*s["args"])
        assert _digest(im) == tuple(s["digest"])
        src.append(im)
    for c in g["crops"]:
        random.seed(c["seed"])
        a = IU.var_center_crop(src[c["src"]], crop_size_list=IU.generate_crop_size_list((512 // 32) ** 2, 32))
        random.seed(c["seed"])
        b = IU.center_crop(src[c["src"]], (256, 128))
        assert _digest(a) == tuple(c["var"]) and _digest(b) == tuple(c["center"])


def test_preprocess_matches_oracle_restatement():
    from mmada_parallel_b200.utils import image_utils as IU
    g = load_golden("amused_glue.pt")
    for im, ind in zip(glue_images(g), g["indices"]):
        x = IU.vae_preprocess(im, 16)
        assert torch.equal(x, AM.preprocess(im, 16))
        assert x.dtype == torch.float32 and tuple(x.shape[2:]) == (ind["Hp"], ind["Wp"])
    x = torch.rand(2, 3, 8, 8)
    assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(IU.vae_postprocess(x), AM.postprocess(x)))


def test_break_and_paint_tokens_match_reference():
    """Token layout with the VQ ids of the fixture: BOI / rows + NEWLINE / EOI for the conditioning image; MASK / code +
    offset / NEWLINE for inpainting and outpainting with every downsample mode and dilation; the visualisation image."""
    from mmada_parallel_b200.utils import image_utils as IU
    g = load_golden("amused_glue.pt")
    for ind, want in zip(g["indices"], g["breaks"]):
        h, w = ind["lat_h"], ind["lat_w"]
        got = [IU.BOI_TOKEN_ID] + IU.add_break_line((ind["ids"] + IU.VQ_OFFSET).tolist(), h, w, IU.NEWLINE_TOKEN_ID) + [IU.EOI_TOKEN_ID]
        assert got == want
    n_masked = 0
    images = glue_images(g)
    for case in g["paint"]:
        kw = dict(case["kwargs"])
        im = images[case["image"]]
        ind = g["indices"][case["image"]]
        W, H = im.size
        cells = IU.paint_latent_mask(W, H, ind["Hp"], ind["Wp"], ind["lat_h"], ind["lat_w"], mask_h_ratio=kw["mask_h_ratio"],
                                     mask_w_ratio=kw["mask_w_ratio"], downsample_mode=kw["downsample_mode"],
                                     dilate_latent_k=kw["dilate_latent_k"], mask_mode=kw["mask_mode"])
        assert IU.paint_tokens(ind["ids"], cells) == case["tokens"].tolist(), kw
        vis = IU.paint_visualisation(im, IU.paint_rect(W, H, kw["mask_h_ratio"], kw["mask_w_ratio"]), kw["gray_value"], kw["mask_mode"])
        assert _digest(vis) == tuple(case["vis"]), kw
        n_masked += int(cells.sum())
    assert n_masked > 0
