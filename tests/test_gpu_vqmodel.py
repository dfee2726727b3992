"""The native aMUSEd VQ-VAE (mmada_parallel_b200.vqmodel.VQModel, variant A's tokenizer) on the H100 against the CPU fp32
oracle (oracle/amused.py, restated from diffusers' structure) and against the reference's own glue
(tests/golden/amused_glue.pt, recorded from the REAL A/utils/image_utils.py over the oracle).

Floating-point tolerances, stated:
  - decode / encode: TF32 products (10-bit mantissa) through ~30-60 convolutions with GroupNorm in between, the MagViT
    bound: per-value |err| <= 0.02 and mean |err| <= 0.003 on outputs with std ~0.6 (the tests print the measured errors);
  - nearest code: exact fp32 distances, so the chosen code equals the fp64 argmin wherever the fp64 gap between the best
    and second-best code exceeds tol = 1e-5 (|z|^2 + max_k |e_k|^2), and is within tol of the minimum everywhere;
  - encode -> quantize: a code may differ only where the latents moved. With z_n the native and z_r the oracle latents, e_n
    and e_r the codes they chose: |z_r - e_n| <= |z_n - e_n| + |z_n - z_r| <= |z_n - e_r| + |z_n - z_r| <= |z_r - e_r| +
    2 |z_n - z_r| (triangle inequality, e_n optimal for z_n); 1e-5 |z_r| covers fp32 rounding. No tuned constant."""
import json

import numpy as np
import pytest
import torch

from helpers import GpuBackedOracleModel, load_golden, tiny_gpu_model
from oracle import amused as AM
from oracle import generate as G
from test_amused_oracle import glue_images

pytestmark = pytest.mark.gpu


def _model(cfg_kw, w, max_batch=1, max_latent_cells=1024):
    from mmada_parallel_b200.vqmodel import VQModel
    L = len(cfg_kw.get("block_out_channels", AM.AMUSED_CONFIG["block_out_channels"]))
    kw = dict(AM.AMUSED_CONFIG, **cfg_kw)
    kw.update(down_block_types=("DownEncoderBlock2D",) * L, up_block_types=("UpDecoderBlock2D",) * L, lookup_from_codebook=True)
    m = VQModel(**kw, max_batch=max_batch, max_latent_cells=max_latent_cells)
    m.load_state_dict(w)
    return m, kw


def _tags():
    return ["small_attn", "small_noattn", "full"]


@pytest.mark.parametrize("tag", _tags())
def test_decode_vs_oracle(tag):
    g = load_golden("amused_vq.pt")[tag]
    cfg = AM.make_config(**g["cfg"])
    w = AM.make_weights(cfg, g["weight_seed"])
    mb = max(r["batch"] for r in g["runs"])
    m, _ = _model(g["cfg"], w, max_batch=mb)
    for run in g["runs"]:
        b, h, wd = run["batch"], run["h"], run["w"]
        ids = run["ids"].cuda()
        out = m.decode(ids, force_not_quantize=True, shape=(b, h, wd, cfg.latent_channels)).sample
        assert tuple(out.shape) == tuple(run["shape"]) and out.dtype == torch.float32
        s = run["stride"]
        err = (out[:, :, ::s, ::s].cpu() - run["image"]).abs()
        print(f"[amused decode {tag} {b}x{h}x{wd}] max err {err.max():.4f} mean err {err.mean():.5f} (image std {run['std']:.3f})")
        assert torch.isfinite(out).all()
        assert err.max() <= 0.02 and err.mean() <= 0.003
        assert abs(float(out.mean()) - run["mean"]) < 5e-3 and abs(float(out.std()) - run["std"]) < 5e-3
        # determinism, and the latents branch gives the same bits as the codebook-lookup branch
        assert torch.equal(m.decode(ids, force_not_quantize=True, shape=(b, h, wd, cfg.latent_channels)).sample, out)
        zq = AM.get_codebook_entry(run["ids"], w, (b, h, wd, cfg.latent_channels)).cuda()
        m.config["lookup_from_codebook"] = False
        try:
            assert torch.equal(m.decode(zq, force_not_quantize=True).sample, out)
        finally:
            m.config["lookup_from_codebook"] = True
        if b > 1:  # batch-row independence
            one = m.decode(ids[1:2], force_not_quantize=True, shape=(1, h, wd, cfg.latent_channels)).sample
            assert torch.allclose(one, out[1:2], atol=1e-5)


@pytest.mark.parametrize("tag", _tags())
def test_encode_and_quantize_vs_oracle(tag):
    g = load_golden("amused_vq.pt")[tag]
    cfg = AM.make_config(**g["cfg"])
    w = AM.make_weights(cfg, g["weight_seed"])
    emb = w["quantize.embedding.weight"].double()
    mb = max(r["batch"] for r in g["runs"])
    m, _ = _model(g["cfg"], w, max_batch=mb)
    scale = 2 ** (len(cfg.block_out_channels) - 1)
    for run in g["runs"]:
        b, h, wd = run["batch"], run["h"], run["w"]
        px = torch.rand(b, 3, h * scale, wd * scale, generator=torch.Generator().manual_seed(run["pixel_seed"]))
        lat = m.encode(px.cuda()).latents
        ls = run["lat_stride"]  # the fixture keeps latent rows 0, ls, 2 ls, ...
        assert lat[:, :, ::ls].shape == run["latents"].shape
        err = (lat[:, :, ::ls].cpu() - run["latents"]).abs()
        print(f"[amused encode {tag} {b}x{h}x{wd}] max err {err.max():.4f} mean err {err.mean():.5f} "
              f"(latent std {float(run['latents'].std()):.3f})")
        assert err.max() <= 0.02 and err.mean() <= 0.003
        assert torch.equal(m.encode(px.cuda()).latents, lat)

        # nearest-code kernel on the oracle's own latents
        z_r = run["latents"].permute(0, 2, 3, 1).reshape(-1, cfg.latent_channels).double()
        d = torch.cdist(z_r, emb) ** 2
        top2 = d.topk(2, largest=False)
        tol = 1e-5 * ((z_r ** 2).sum(1) + (emb ** 2).sum(1).max())
        zq, _, (_, _, ids) = m.quantize(run["latents"].cuda())
        ids = ids.cpu()
        decided = (top2.values[:, 1] - top2.values[:, 0]) > tol
        assert torch.equal(ids[decided], run["quant_ids"][decided])
        chosen = d.gather(1, ids[:, None])[:, 0]
        assert (chosen - top2.values[:, 0] <= tol).all()
        hs = run["latents"].shape[2]
        assert torch.equal(zq.cpu(), w["quantize.embedding.weight"][ids].view(b, hs, wd, -1).permute(0, 3, 1, 2))
        print(f"[amused quantize {tag}] decided {int(decided.sum())}/{len(ids)}, equal "
              f"{int((ids == run['quant_ids']).sum())}/{len(ids)}")

        # end to end: encode -> quantize
        _, _, (_, _, ids_n) = m.quantize(lat)
        ids_n = ids_n.view(b, h, wd)[:, ::ls].reshape(-1)
        z_n = lat[:, :, ::ls].permute(0, 2, 3, 1).reshape(-1, cfg.latent_channels).double().cpu()
        e_n, e_r = emb[ids_n.cpu()], emb[run["quant_ids"]]
        lhs = (z_r - e_n).norm(dim=1)
        rhs = (z_r - e_r).norm(dim=1) + 2 * (z_n - z_r).norm(dim=1) + 1e-5 * z_r.norm(dim=1)
        assert (lhs <= rhs).all()


def _glue_model():
    g = load_golden("amused_glue.pt")
    cfg = AM.make_config(**g["cfg"])
    w = AM.make_weights(cfg, g["weight_seed"])
    m, kw = _model(g["cfg"], w, max_latent_cells=384)
    return g, cfg, w, m, kw


def _tokens_within_bound(got, want, m, w, cfg, img):
    """Token lists equal except at codes the encode -> quantize bound allows (module docstring)."""
    assert len(got) == len(want)
    diff = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    if not diff:
        return 0
    from mmada_parallel_b200.utils import image_utils as IU
    x = IU.vae_preprocess(img, 2 ** (len(cfg.block_out_channels) - 1))
    z_n = m.encode(x.cuda()).latents.cpu()
    z_r = AM.encode(x, w, cfg)
    lw = z_r.shape[3]
    emb = w["quantize.embedding.weight"].double()
    for i in diff:
        a, b = got[i], want[i]
        assert IU.VQ_OFFSET <= a < IU.VQ_OFFSET + cfg.num_vq_embeddings and IU.VQ_OFFSET <= b < IU.VQ_OFFSET + cfg.num_vq_embeddings
        # position i in a row-major list with a NEWLINE after every row (and a leading BOI for the conditioning image)
        k = i - 1 if want[0] == IU.BOI_TOKEN_ID else i
        y, x_ = divmod(k, lw + 1)
        zr, zn = z_r[0, :, y, x_].double(), z_n[0, :, y, x_].double()
        lhs = (zr - emb[a - IU.VQ_OFFSET]).norm()
        rhs = (zr - emb[b - IU.VQ_OFFSET]).norm() + 2 * (zn - zr).norm() + 1e-5 * zr.norm()
        assert lhs <= rhs, (i, a, b)
    return len(diff)


def test_glue_vs_reference():
    from mmada_parallel_b200.utils import image_utils as IU
    g, cfg, w, m, _ = _glue_model()
    for case in g["decode"]:
        img = IU.decode_vq_to_image(case["ids"].cuda(), None, None, case["height"], case["width"], m)
        got = np.asarray(img).astype(int)
        want = case["image"].astype(int)
        assert got.shape == want.shape
        d = np.abs(got - want)
        print(f"[glue decode {case['height']}x{case['width']}] max level diff {d.max()}, share > 1: {(d > 1).mean():.5f}, "
              f"share > 0: {(d > 0).mean():.4f}")
        assert (d > 1).mean() <= 1e-3
    n_diff = 0
    images = glue_images(g)
    for im, want in zip(images, g["breaks"]):
        n_diff += _tokens_within_bound(IU.encode_img_with_breaks(im, m), want, m, w, cfg, im)
    for case in g["paint"]:
        im = images[case["image"]]
        want = case["tokens"].tolist()
        tokens, _ = IU.encode_img_with_paint(im, m, **case["kwargs"])
        assert [t == IU.MASK_TOKEN_ID for t in tokens] == [t == IU.MASK_TOKEN_ID for t in want]
        n_diff += _tokens_within_bound(tokens, want, m, w, cfg, im)
    print(f"[glue tokens] {n_diff} codes differ from the reference glue, all within the bound")


def test_stepwise_preview_with_vqmodel():
    """generate_ti2ti_stepwise's preview helpers read the scale of a VQModel from its config."""
    from mmada_parallel_b200.utils.image_utils import decode_vq_to_image, vq_scale
    g, cfg, _, m, _ = _glue_model()
    assert vq_scale(m) == 16
    case = g["decode"][1]
    img = decode_vq_to_image(case["ids"].cuda(), None, None, case["height"], case["width"], m)
    assert img.size == (case["width"], case["height"])


def test_from_pretrained_bit_identical(tmp_path):
    from safetensors.torch import save_file
    from mmada_parallel_b200.utils.image_utils import decode_vq_to_image
    from mmada_parallel_b200.vqmodel import VQModel
    g, cfg, w, m, kw = _glue_model()
    d = tmp_path / "ckpt" / "vqvae"
    d.mkdir(parents=True)
    conf = {k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()}
    conf.update(_class_name="VQModel", _diffusers_version="0.34.0", sample_size=32, scaling_factor=0.18215, force_upcast=False,
                norm_type="group", act_fn="silu", vq_embed_dim=None)
    (d / "config.json").write_text(json.dumps(conf))
    # deprecated attention names in the file: load_state_dict maps them
    sd = {k.replace(".to_q.", ".query.").replace(".to_out.0.", ".proj_attn."): v.contiguous() for k, v in w.items()}
    save_file(sd, str(d / "diffusion_pytorch_model.safetensors"))
    m2 = VQModel.from_pretrained(str(tmp_path / "ckpt"), subfolder="vqvae", max_latent_cells=384)
    case = g["decode"][1]
    ids, hh, ww = case["ids"].cuda(), case["height"], case["width"]
    shape = (1, hh // 16, ww // 16, cfg.latent_channels)
    a = m.decode(ids.view(shape[:3]), force_not_quantize=True, shape=shape).sample
    b = m2.decode(ids.view(shape[:3]), force_not_quantize=True, shape=shape).sample
    assert torch.equal(a, b)
    x = torch.rand(1, 3, 64, 96, generator=torch.Generator().manual_seed(0)).cuda()
    assert torch.equal(m.encode(x).latents, m2.encode(x).latents)
    # decode_vq_to_image loads <vae_ckpt>/vqvae when no model is passed
    img = decode_vq_to_image(ids, None, str(tmp_path / "ckpt"), hh, ww, None)
    assert np.array_equal(np.asarray(img), np.asarray(decode_vq_to_image(ids, None, None, hh, ww, m)))


def test_errors():
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.utils.image_utils import decode_vq_to_image
    from mmada_parallel_b200.vqmodel import VQModel
    g, cfg, w, m, kw = _glue_model()
    fresh = VQModel(**kw, max_latent_cells=64)
    with pytest.raises(_lib.MmdpError, match="not loaded"):
        fresh.decode(torch.zeros(1, 4, 4, dtype=torch.long).cuda(), force_not_quantize=True, shape=(1, 4, 4, cfg.latent_channels))
    with pytest.raises(RuntimeError):
        fresh.load_state_dict({k: v for k, v in w.items() if "conv_out" not in k})
    with pytest.raises(ValueError):  # grid over max_latent_cells
        m.decode(torch.zeros(1, 20, 20, dtype=torch.long).cuda(), force_not_quantize=True, shape=(1, 20, 20, cfg.latent_channels))
    with pytest.raises(ValueError):
        m.encode(torch.zeros(1, 3, 320, 320).cuda())
    with pytest.raises(ValueError):  # length mismatch
        decode_vq_to_image(torch.zeros(1, 250, dtype=torch.long).cuda(), None, None, 256, 256, m)
    with pytest.raises(IndexError):  # id outside the codebook
        m.decode(torch.full((1, 4, 4), cfg.num_vq_embeddings, dtype=torch.long).cuda(), force_not_quantize=True,
                 shape=(1, 4, 4, cfg.latent_channels))
    m.decode(torch.zeros(1, 4, 4, dtype=torch.long).cuda(), force_not_quantize=True, shape=(1, 4, 4, cfg.latent_channels))  # flag cleared
    with pytest.raises(ValueError):  # bad config
        VQModel(**dict(kw, norm_num_groups=16))
    # the C layer refuses what the Python layer would have caught
    import ctypes as C
    c = _lib.VqModelConfig()
    c.in_channels, c.out_channels, c.n_levels, c.layers_per_block, c.latent_channels = 3, 3, 2, 1, 300
    c.block_out_channels[0], c.block_out_channels[1] = 32, 64
    c.num_vq_embeddings, c.max_batch, c.max_latent_cells = 16, 1, 16
    h = C.c_void_p()
    assert _lib.lib.mmdp_vqmodel_create(C.byref(c), C.byref(h)) == -1 and b"latent_channels" in _lib.lib.mmdp_last_error()
    c.latent_channels, c.block_out_channels[1] = 16, 48
    assert _lib.lib.mmdp_vqmodel_create(C.byref(c), C.byref(h)) == -1 and b"multiple of 32" in _lib.lib.mmdp_last_error()


def test_painting_mode_lockstep_with_oracle():
    """Inpainting / outpainting inputs (built by the reference glue): the product loop equals the oracle loop on identical
    logits, and the known image tokens are never changed."""
    import contextlib
    import io
    from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti
    t = load_golden("trajectory_paint_tiny.pt")
    model, _, _ = tiny_gpu_model(t["meta"])
    backed = GpuBackedOracleModel(model)
    for run in t["runs"]:
        lay = run["layout"]
        args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
        torch.manual_seed(run["global_seed"])
        img_o, txt_o = G.generate_ti2ti(backed, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]),
                                        stable_sort=True, **args, **run["kwargs"])
        torch.manual_seed(run["global_seed"])
        with contextlib.redirect_stdout(io.StringIO()):
            img_g, txt_g = generate_ti2ti(model, lay["input_ids"], generator=torch.Generator().manual_seed(run["seed"]), **args,
                                          **run["kwargs"])
        assert img_g == img_o and txt_g == txt_o, run["name"]
        # known cells keep their code: the image span of the input without its NEWLINEs
        span = lay["input_ids"][0, lay["image_start"]:lay["image_start"] + lay["seq_len"] + lay["seq_len"] // lay["newline_every"]]
        known = [int(v) - 126356 for v in span if int(v) not in (126084, 126336)]
        cells = [int(v) for v in span if int(v) != 126084]
        assert len(cells) == lay["seq_len"] and known
        for i, v in enumerate(cells):
            if v != 126336:
                assert img_g[i] == v - 126356, (run["name"], i)
                assert run["image_tokens"][i] == v - 126356, (run["name"], i)
