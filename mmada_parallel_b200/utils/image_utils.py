"""Drop-in for `decode_vq_to_image` (MMaDA-Parallel-A/utils/image_utils.py:13-75): VQ ids -> PIL image.

The reference decodes with the aMUSEd VQ-VAE (`diffusers.VQModel`, not part of this repository - DESIGN.md section 5); here
the decoder is any object with the native protocol of `mmada_parallel_b200.magvit.MAGVITv2`:
    vqvae.decode_code(ids[B, N]) -> FloatTensor[B, 3, H, W] in ~[-1, 1]      (C call into the TF32 wgmma decoder)
    vqvae.decoder.upscale                                                     (pixels per latent cell, 16 for 5 levels)
Same arguments, same `ValueError` on a length mismatch (:48-52), same return type (one PIL image, batch row 0).
"""
from __future__ import annotations

from typing import List, Optional

import torch
from PIL import Image, ImageDraw


def vq_scale(vqvae) -> int:
    dec = getattr(vqvae, "decoder", None)
    scale = getattr(dec, "upscale", None) or getattr(vqvae, "upscale", None)
    if scale is None or not hasattr(vqvae, "decode_code"):
        raise TypeError("decode_vq_to_image needs a native VQ decoder (mmada_parallel_b200.magvit.MAGVITv2 protocol: "
                        ".decode_code(ids) and .decoder.upscale); the diffusers VQModel route of the reference is not built")
    return int(scale)


def decode_vq_to_image(vq_codes: torch.Tensor, save_path: Optional[str] = None, vae_ckpt: Optional[str] = None,
                       image_height: int = 512, image_width: int = 512, vqvae=None) -> Image.Image:
    if vqvae is None:
        raise ValueError("decode_vq_to_image: pass vqvae= (loading the aMUSEd VQ-VAE from vae_ckpt needs diffusers, which this "
                         "repository does not use)")
    scale = vq_scale(vqvae)
    latent_h, latent_w = image_height // scale, image_width // scale
    expected_len = latent_h * latent_w
    if vq_codes.shape[1] != expected_len:
        raise ValueError(f"VQ codes length mismatch: {vq_codes.shape[1]} != {expected_len} "
                         f"for image size ({image_height},{image_width}) with scale {scale}")
    recon = vqvae.decode_code(vq_codes.long(), shape=(latent_h, latent_w))          # [B, 3, H, W], ~[-1, 1]
    recon = ((recon[0] + 1.0) * 0.5).clamp(0, 1)                                     # M/inference.py:129 convention
    arr = (recon.permute(1, 2, 0) * 255.0).round().to(torch.uint8).cpu().numpy()    # VaeImageProcessor.numpy_to_pil rounding
    img = Image.fromarray(arr)
    if save_path is not None:
        img.save(save_path)
    return img


def overlay_masked_cells(img: Image.Image, masked_idx: List[int], token_w: int, pixel_h: int, pixel_w: int) -> Image.Image:
    """Grey translucent squares over still-masked latent cells (A/app.py:312-333, :377-396)."""
    img = img.copy()
    draw = ImageDraw.Draw(img, "RGBA")
    for i in masked_idx:
        y1, x1 = (i // token_w) * pixel_h, (i % token_w) * pixel_w
        draw.rectangle([x1, y1, x1 + pixel_w, y1 + pixel_h], fill=(128, 128, 128, 120))
    return img
