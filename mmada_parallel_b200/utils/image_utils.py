"""Variant A's image glue (MMaDA-Parallel-A/utils/image_utils.py): VQ ids -> PIL image, and PIL image -> the id lists the
denoising loop conditions on, including the inpainting / outpainting inputs of A/inference.py:141-146.

Two decoder protocols are accepted by `decode_vq_to_image`:
  - the aMUSEd VQ-VAE, `mmada_parallel_b200.vqmodel.VQModel` (variant A's tokenizer; anything with
    `config.block_out_channels`, as the reference detects it): `.decode(ids, force_not_quantize=True, shape=(B, h, w, C))`,
    `.sample.clip(0, 1)`, then VaeImageProcessor.postprocess without normalisation: (x * 255).round() -> uint8;
  - the native MagViT protocol of `mmada_parallel_b200.magvit.MAGVITv2` (variant M's tokenizer):
    `vqvae.decode_code(ids[B, N]) -> FloatTensor[B, 3, H, W]` in ~[-1, 1] and `vqvae.decoder.upscale`.
Same arguments, same `ValueError` on a length mismatch (:48-52), same return type (one PIL image, batch row 0).
"""
from __future__ import annotations

import random
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image, ImageDraw

# token ids of variant A's vocabulary (A/utils/image_utils.py:169-172, :210-212)
MASK_TOKEN_ID = 126336
NEWLINE_TOKEN_ID = 126084
VQ_OFFSET = 126356
BOI_TOKEN_ID = 126349
EOI_TOKEN_ID = 126350


def _is_vqmodel(vqvae) -> bool:
    return getattr(getattr(vqvae, "config", None), "block_out_channels", None) is not None


def vq_scale(vqvae) -> int:
    """Pixels per latent cell of a decoder of either protocol."""
    if _is_vqmodel(vqvae):
        return 2 ** (len(vqvae.config.block_out_channels) - 1)
    dec = getattr(vqvae, "decoder", None)
    scale = getattr(dec, "upscale", None) or getattr(vqvae, "upscale", None)
    if scale is None or not hasattr(vqvae, "decode_code"):
        raise TypeError("decode_vq_to_image needs a native VQ decoder: mmada_parallel_b200.vqmodel.VQModel (aMUSEd, "
                        ".config.block_out_channels) or the mmada_parallel_b200.magvit.MAGVITv2 protocol (.decode_code(ids) and "
                        ".decoder.upscale)")
    return int(scale)


# ---- VaeImageProcessor(vae_scale_factor, do_normalize=False) ---------------------------------------------------------
def vae_preprocess(img: Image.Image, vae_scale_factor: int) -> torch.Tensor:
    """VaeImageProcessor.preprocess without normalisation: resize to multiples of the scale factor (PIL Lanczos), then
    /255 to fp32 NCHW [1, 3, H, W] in [0, 1]."""
    w, h = img.size
    w, h = w - w % vae_scale_factor, h - h % vae_scale_factor
    img = img.resize((w, h), resample=Image.LANCZOS)
    arr = np.asarray(img.convert("RGB"), dtype=np.float32) / 255.0
    return torch.from_numpy(arr[None]).permute(0, 3, 1, 2).contiguous()


def vae_postprocess(x: torch.Tensor) -> List[Image.Image]:
    """VaeImageProcessor.postprocess(output_type="pil") without denormalisation: (x * 255).round() -> uint8."""
    arr = x.detach().float().cpu().permute(0, 2, 3, 1).numpy()
    return [Image.fromarray(a) for a in (arr * 255).round().astype("uint8")]


def decode_vq_to_image(vq_codes: torch.Tensor, save_path: Optional[str] = None, vae_ckpt: Optional[str] = None,
                       image_height: int = 512, image_width: int = 512, vqvae=None) -> Image.Image:
    if vqvae is None:
        if vae_ckpt is None:
            raise ValueError("decode_vq_to_image: pass vqvae= or vae_ckpt= (a local diffusers directory with a vqvae/ subfolder)")
        from ..vqmodel import VQModel
        dev = vq_codes.device if vq_codes.is_cuda else "cuda:0"
        vqvae = VQModel.from_pretrained(vae_ckpt, subfolder="vqvae", device=dev)
    scale = vq_scale(vqvae)
    latent_h, latent_w = image_height // scale, image_width // scale
    expected_len = latent_h * latent_w
    if vq_codes.shape[1] != expected_len:
        raise ValueError(f"VQ codes length mismatch: {vq_codes.shape[1]} != {expected_len} "
                         f"for image size ({image_height},{image_width}) with scale {scale}")
    if _is_vqmodel(vqvae):
        b = vq_codes.shape[0]
        lat = vq_codes.reshape(b, latent_h, latent_w).long()
        recon = vqvae.decode(lat, force_not_quantize=True, shape=(b, latent_h, latent_w, vqvae.config.latent_channels)).sample
        img = vae_postprocess(recon.clip(0, 1))[0]
    else:
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


# ---- layout helpers ----------------------------------------------------------------------------------------------
def calculate_vq_params(image_height: int, image_width: int, vae_scale: int = 16) -> Tuple[int, int, int, int]:
    """(seq_len, newline_every, token_grid_height, token_grid_width) of an output image."""
    gh, gw = image_height // vae_scale, image_width // vae_scale
    return gh * gw, gw, gh, gw


def add_break_line(sequence: list, H: int, W: int, new_number: int = 0) -> list:
    """Row-major H x W ids with `new_number` appended after every row."""
    out = []
    for r in range(H):
        out += list(sequence[r * W:(r + 1) * W])
        out.append(new_number)
    return out


def generate_crop_size_list(num_patches: int, patch_size: int, max_ratio: float = 4.0) -> List[Tuple[int, int]]:
    """(width, height) pairs of at most num_patches patches with aspect ratio <= max_ratio: the width in patches walks down
    from num_patches while the height grows as far as the patch budget allows."""
    assert max_ratio >= 1.0
    sizes = []
    wp, hp = num_patches, 1
    while wp > 0:
        if max(wp, hp) / min(wp, hp) <= max_ratio:
            sizes.append((wp * patch_size, hp * patch_size))
        if wp * (hp + 1) <= num_patches:
            hp += 1
        else:
            wp -= 1
    return sizes


def center_crop(pil_image: Image.Image, crop_size: Tuple[int, int]) -> Image.Image:
    """Halve with BOX while the image is at least twice the crop, scale with BICUBIC so the crop just fits, then crop at
    a position drawn from Python's `random` (uniform over the valid offsets)."""
    cw, ch = crop_size
    while pil_image.size[0] >= 2 * cw and pil_image.size[1] >= 2 * ch:
        pil_image = pil_image.resize(tuple(v // 2 for v in pil_image.size), resample=Image.BOX)
    s = max(cw / pil_image.size[0], ch / pil_image.size[1])
    pil_image = pil_image.resize(tuple(round(v * s) for v in pil_image.size), resample=Image.BICUBIC)
    left = random.randint(0, pil_image.size[0] - cw)
    top = random.randint(0, pil_image.size[1] - ch)
    return pil_image.crop(box=(left, top, left + cw, top + ch))


def var_center_crop(pil_image: Image.Image, crop_size_list, random_top_k: int = 1) -> Image.Image:
    """Center-crop to the listed size whose aspect ratio is closest to the image's (one of the random_top_k closest)."""
    w, h = pil_image.size
    ranked = sorted(((min(cw / w, ch / h) / max(cw / w, ch / h), (cw, ch)) for cw, ch in crop_size_list), reverse=True)
    return center_crop(pil_image, random.choice(ranked[:random_top_k])[1])


def preprocess_image(image_path: str, target_size: tuple = (512, 512)) -> Image.Image:
    img = Image.open(image_path).convert("RGB")
    return var_center_crop(img, crop_size_list=generate_crop_size_list((target_size[0] // 32) ** 2, 32))


# ---- encode ------------------------------------------------------------------------------------------------------
def _encode_indices(img: Image.Image, vqvae, vae_scale_factor: int):
    x = vae_preprocess(img, vae_scale_factor).to(vqvae.device)
    lat = vqvae.encode(x).latents
    b, _, h, w = lat.shape
    ids = vqvae.quantize(lat)[2][2]
    return x, ids.reshape(b, h, w), h, w


@torch.no_grad()
def encode_img_with_breaks(img: Image.Image, vqvae, vae_scale_factor: int = 16) -> List[int]:
    """[BOI] + rows of (code + VQ_OFFSET) each followed by NEWLINE + [EOI]: the conditioning image of A/inference.py:127."""
    _, ids, h, w = _encode_indices(img.convert("RGB"), vqvae, vae_scale_factor)
    codes = (ids + VQ_OFFSET).flatten().tolist()
    return [BOI_TOKEN_ID] + add_break_line(codes, h, w, new_number=NEWLINE_TOKEN_ID) + [EOI_TOKEN_ID]


def paint_rect(W: int, H: int, mask_h_ratio: float, mask_w_ratio: float) -> Tuple[int, int, int, int]:
    """(left, top, right, bottom) of the centred mask rectangle of an image W x H pixels."""
    mh, mw = int(round(H * mask_h_ratio)), int(round(W * mask_w_ratio))
    top, left = (H - mh) // 2, (W - mw) // 2
    return left, top, left + mw, top + mh


def paint_latent_mask(W: int, H: int, Hp: int, Wp: int, lat_h: int, lat_w: int, *, mask_h_ratio: float, mask_w_ratio: float,
                      downsample_mode: str = "area", dilate_latent_k: int = 0, mask_mode: str = "inpainting") -> torch.Tensor:
    """Latent cells to mask (bool [lat_h, lat_w]) for an image of W x H pixels encoded at Wp x Hp: the centred rectangle is
    mapped to the encoder's pixel grid, inverted for outpainting, resampled to the latent grid (`area`: mean > 0.5;
    `nearest` / `bilinear`: >= 0.5; any other mode means `area`) and optionally dilated by a (2k+1)^2 max filter."""
    left, top, right, bottom = paint_rect(W, H, mask_h_ratio, mask_w_ratio)
    mh, mw = bottom - top, right - left
    m = torch.zeros((1, 1, Hp, Wp), dtype=torch.float32)
    tp, lp = int(round(top * Hp / H)), int(round(left * Wp / W))
    hp, wp = int(round(mh * Hp / H)), int(round(mw * Wp / W))
    m[:, :, tp:tp + hp, lp:lp + wp] = 1.0
    if mask_mode == "outpainting":
        m = 1.0 - m
    if downsample_mode not in ("nearest", "area", "bilinear"):
        downsample_mode = "area"
    m = F.interpolate(m, size=(lat_h, lat_w), mode=downsample_mode)
    cells = m > 0.5 if downsample_mode == "area" else m >= 0.5
    if dilate_latent_k > 0:
        k = dilate_latent_k
        cells = F.max_pool2d(cells.float(), kernel_size=2 * k + 1, stride=1, padding=k) > 0.5
    return cells[0, 0]


def paint_tokens(indices: torch.Tensor, cell_mask: torch.Tensor) -> List[int]:
    """Row-major tokens of a latent grid: MASK where cell_mask, code + VQ_OFFSET elsewhere, NEWLINE after every row."""
    lat_h, lat_w = cell_mask.shape
    idx = indices.reshape(-1).cpu()
    tokens = torch.where(cell_mask.reshape(-1).cpu(), torch.full_like(idx, MASK_TOKEN_ID), idx + VQ_OFFSET)
    return add_break_line(tokens.tolist(), lat_h, lat_w, NEWLINE_TOKEN_ID)


def paint_visualisation(img: Image.Image, rect, gray_value: int, mask_mode: str) -> Image.Image:
    left, top, right, bottom = rect
    g = (gray_value, gray_value, gray_value)
    if mask_mode == "inpainting":
        vis = img.copy()
        ImageDraw.Draw(vis).rectangle([left, top, right, bottom], fill=g)
        return vis
    vis = Image.new("RGB", img.size, g)
    vis.paste(img.crop((left, top, right, bottom)), (left, top))
    return vis


@torch.no_grad()
def encode_img_with_paint(img: Image.Image, vqvae, *, mask_h_ratio: float = 1, mask_w_ratio: float = 0.2, gray_value: int = 127,
                          downsample_mode: str = "area", dilate_latent_k: int = 0, mask_mode: str = "inpainting"):
    """Inpainting / outpainting input (A/inference.py:141-146): the whole image is encoded, and the latent cells under the
    centred rectangle (inpainting) or outside it (outpainting) become MASK tokens. Returns (tokens with a NEWLINE after
    every row and no BOI / EOI, grey visualisation image)."""
    assert mask_mode in ("inpainting", "outpainting"), "mask_mode must be 'inpainting' or 'outpainting'"
    img = img.convert("RGB")
    W, H = img.size
    vis = paint_visualisation(img, paint_rect(W, H, mask_h_ratio, mask_w_ratio), gray_value, mask_mode)
    x, ids, lat_h, lat_w = _encode_indices(img, vqvae, vq_scale(vqvae))
    Hp, Wp = x.shape[-2:]
    cells = paint_latent_mask(W, H, Hp, Wp, lat_h, lat_w, mask_h_ratio=mask_h_ratio, mask_w_ratio=mask_w_ratio,
                              downsample_mode=downsample_mode, dilate_latent_k=dilate_latent_k, mask_mode=mask_mode)
    return paint_tokens(ids[0], cells), vis
