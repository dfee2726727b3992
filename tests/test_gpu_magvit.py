"""MAGVITv2.decode_code on the H100 (TF32 wgmma convolutions) against the golden images produced by the REAL
reference decoder (fp32, CPU; oracle pinned bit-exact in oracle/make_golden_magvit.py).
Floating-point tolerance (stated): TF32 products (10-bit mantissa) through ~35 convolutions with GroupNorm in between;
per-pixel |err| <= 0.02 and mean |err| <= 0.003 on images with std ~0.55, |max| ~3.4 (the test prints the measured errors;
one 8-bit pixel step is 1/127.5 = 0.0078 after the caller's (x+1)/2 mapping).
Deviation from torch's defaults, stated: every contraction of the decoder runs with TF32 products, including the two
matmuls of the mid-block AttnBlock; torch.backends.cuda.matmul.allow_tf32 defaults to False (fp32 matmul) while cuDNN
convolutions default to TF32, so the reference on a GPU would run those two matmuls in fp32 - 2 of ~60 contractions,
inside the bound above."""
import pytest
import torch

from helpers import load_golden
from oracle import magvit as OM

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag", ["small", "full"])
def test_decode_code_vs_reference_golden(tag):
    from mmada_parallel_b200.magvit import MAGVITv2
    g = load_golden("magvit_decode.pt")[tag]
    cfg = OM.decoder_config(**g["cfg"])
    w = OM.make_weights(cfg, g["weight_seed"])
    idx = g["idx"]
    hw = int(idx.shape[1] ** 0.5)
    m = MAGVITv2(max_batch=idx.shape[0], ch=cfg.ch, ch_mult=cfg.ch_mult, num_res_blocks=cfg.num_res_blocks, latent_hw=(hw, hw))
    m.load_state_dict(w)
    out = m.decode_code(idx)
    assert tuple(out.shape) == tuple(g["shape"]) and out.dtype == torch.float32
    s = g["stride"]
    got = out[:, :, ::s, ::s].cpu()
    err = (got - g["image"]).abs()
    print(f"[magvit {tag}] max err {err.max():.4f} mean err {err.mean():.5f} (image std {g['std']:.3f})")
    assert torch.isfinite(out).all()
    assert err.max() <= 0.02 and err.mean() <= 0.003
    assert abs(float(out.mean()) - g["mean"]) < 5e-3 and abs(float(out.std()) - g["std"]) < 5e-3
    # determinism + batch independence
    out2 = m.decode_code(idx)
    assert torch.equal(out, out2)
    if idx.shape[0] > 1:
        m1 = MAGVITv2(max_batch=1, ch=cfg.ch, ch_mult=cfg.ch_mult, num_res_blocks=cfg.num_res_blocks, latent_hw=(hw, hw))
        m1.load_state_dict(w)
        assert torch.allclose(m1.decode_code(idx[1:2]), out[1:2], atol=1e-5)


def test_decode_code_errors():
    from mmada_parallel_b200 import _lib
    from mmada_parallel_b200.magvit import MAGVITv2
    m = MAGVITv2(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 2), latent_hw=(8, 8))
    with pytest.raises(_lib.MmdpError):  # weights not loaded
        m.decode_code(torch.zeros(1, 64, dtype=torch.long))
    with pytest.raises(ValueError):
        m.decode_code(torch.zeros(1, 60, dtype=torch.long))
    with pytest.raises(_lib.MmdpError):  # encoder weights not loaded
        m.get_code(torch.zeros(1, 3, 16, 16))


@pytest.mark.parametrize("tag", ["small", "full"])
def test_get_code_vs_reference_golden(tag):
    """MAGVITv2.get_code: the 13 sign bits of the encoder output. TF32 products perturb the pre-quantisation map by ~1e-3, so a
    bit may flip only where the reference's own value is within that distance of zero: required - every differing bit
    sits on |z_ref| < 0.02 (z has std ~0.5, so a few percent of the 13-bit codes contain such a near-zero channel)."""
    from mmada_parallel_b200.magvit import MAGVITv2
    g = load_golden("magvit_encode.pt")[tag]
    cfg = OM.encoder_config(**g["cfg"])
    w = OM.make_encoder_weights(cfg, g["weight_seed"])
    res, batch = g["res"], g["batch"]
    px = torch.rand(batch, 3, res, res, generator=torch.Generator().manual_seed(g["pixel_seed"])) * 2 - 1
    lat = res // 2 ** (len(cfg.ch_mult) - 1)
    dec_kw = dict(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 1), latent_hw=(lat, lat))  # decoder side unused here
    m = MAGVITv2(max_batch=batch, encoder_kw=dict(ch=cfg.ch, ch_mult=cfg.ch_mult, num_res_blocks=cfg.num_res_blocks), **dec_kw)
    m.load_state_dict(w)
    ids = m.get_code(px).cpu()
    assert ids.shape == g["ids"].shape and ids.dtype == torch.int64
    diff = ids ^ g["ids"]
    frac = (diff != 0).float().mean().item()
    z = g["z"].reshape(batch, 13, -1)
    bad_margin = 0.0
    for bit in range(13):
        flipped = ((diff >> (12 - bit)) & 1).bool()
        if flipped.any():
            bad_margin = max(bad_margin, z[:, bit][flipped].abs().max().item())
    print(f"[magvit get_code {tag}] codes differing {frac:.4f}, largest |z_ref| at a flipped bit {bad_margin:.4f}")
    assert frac < 0.15 and bad_margin < 0.02
    assert torch.equal(m.get_code(px).cpu(), ids)
