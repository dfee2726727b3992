"""ORACLE (test infrastructure, NOT product code): CPU fp32 restatement of the aMUSEd VQ-VAE, `diffusers.VQModel`, the
tokenizer variant A loads in MMaDA-Parallel-A/utils/image_utils.py (decode :13-75, encode :159-173 and :176-285).

RESTATED FROM DIFFUSERS' STRUCTURE, NOT PINNED AGAINST DIFFUSERS: neither diffusers nor the aMUSEd checkpoint is available
where this file was written, so unlike oracle/magvit.py nothing here has been compared with the real modules. Each fact
below names the diffusers 0.34.0 source it restates, so that someone holding diffusers can check it line by line:

  autoencoders/vq_model.py, VQModel
    __init__: encoder = Encoder(in_channels, out_channels=latent_channels, down_block_types, block_out_channels,
              layers_per_block, act_fn, norm_num_groups, double_z=False, mid_block_add_attention);
              vq_embed_dim = vq_embed_dim or latent_channels; quant_conv = Conv2d(latent_channels, vq_embed_dim, 1);
              quantize = VectorQuantizer(num_vq_embeddings, vq_embed_dim, beta=0.25, remap=None, sane_index_shape=False);
              post_quant_conv = Conv2d(vq_embed_dim, latent_channels, 1);
              decoder = Decoder(in_channels=latent_channels, out_channels, up_block_types, block_out_channels,
              layers_per_block, act_fn, norm_num_groups, norm_type, mid_block_add_attention).
    encode(x): h = quant_conv(encoder(x)); returns VQEncoderOutput(latents=h).
    decode(h, force_not_quantize=False, shape=None):
              not force_not_quantize      -> quant, commit_loss, _ = quantize(h)
              elif lookup_from_codebook   -> quant = quantize.get_codebook_entry(h, shape)
              else                        -> quant = h
              dec = decoder(post_quant_conv(quant), quant if norm_type == "spatial" else None); returns .sample.
  autoencoders/vae.py, VectorQuantizer
    forward(z): z -> NHWC, flattened [N, C]; indices = argmin(torch.cdist(z_flat, embedding.weight), dim=1);
              z_q = embedding(indices).view(z.shape); z_q = z + (z_q - z).detach() (straight-through); back to NCHW;
              returns (z_q, loss, (perplexity, min_encodings, indices)) with indices flat in (b, y, x) order.
    get_codebook_entry(indices, shape): z_q = embedding(indices); view(shape) with shape = (B, h, w, C); permute to NCHW.
  autoencoders/vae.py, Encoder.forward
    conv_in (3x3, pad 1, in_channels -> block_out_channels[0]) -> down_blocks.i -> mid_block -> conv_norm_out
    (GroupNorm(norm_num_groups, block_out_channels[-1], eps=1e-6)) -> SiLU -> conv_out (3x3, pad 1, -> latent_channels;
    2 * latent_channels only with double_z). down_blocks.i = DownEncoderBlock2D(num_layers=layers_per_block,
    in=block_out_channels[i-1] (block_out_channels[0] for i = 0), out=block_out_channels[i], resnet_eps=1e-6,
    add_downsample = not is_final_block, downsample_padding=0).
    mid_block = UNetMidBlock2D(block_out_channels[-1], resnet_eps=1e-6, attention_head_dim=block_out_channels[-1],
    resnet_groups=norm_num_groups, temb_channels=None, add_attention=mid_block_add_attention).
  autoencoders/vae.py, Decoder.forward
    conv_in (3x3, pad 1, latent_channels -> block_out_channels[-1]) -> mid_block -> up_blocks.i -> conv_norm_out
    (GroupNorm(norm_num_groups, block_out_channels[0], eps=1e-6)) -> SiLU -> conv_out (3x3, pad 1, -> out_channels).
    up_blocks.i = UpDecoderBlock2D(num_layers=layers_per_block + 1, in=reversed(block_out_channels)[i-1]
    (block_out_channels[-1] for i = 0), out=reversed(block_out_channels)[i], resnet_eps=1e-6,
    add_upsample = not is_final_block).
  unets/unet_2d_blocks.py
    DownEncoderBlock2D: resnets.j = ResnetBlock2D(in if j == 0 else out, out, temb_channels=None);
                        downsamplers.0 = Downsample2D(out, use_conv=True, padding=0, name="op") (parameter `.conv`).
    UpDecoderBlock2D:   resnets.j = ResnetBlock2D(in if j == 0 else out, out, temb_channels=None);
                        upsamplers.0 = Upsample2D(out, use_conv=True) (parameter `.conv`).
    UNetMidBlock2D:     resnets.0 -> attentions.0 (when add_attention) -> resnets.1, both resnets C -> C.
                        attentions.0 = Attention(C, heads=C // attention_head_dim = 1, dim_head=C, eps=resnet_eps,
                        norm_num_groups=resnet_groups, residual_connection=True, bias=True, upcast_softmax=True,
                        _from_deprecated_attn_block=True): group_norm -> to_q / to_k / to_v (Linear [C, C]) ->
                        softmax(q k^T / sqrt(C)) v -> to_out.0 (Linear) -> + residual (rescale_output_factor 1).
                        Checkpoints saved before the rename use query / key / value / proj_attn.
  models/resnet.py, ResnetBlock2D (temb None, output_scale_factor 1, dropout 0)
    h = conv2(SiLU(norm2(conv1(SiLU(norm1(x)))))); x = conv_shortcut(x) (1x1) when in != out; returns x + h.
    norm1 / norm2: GroupNorm(32, eps=1e-6); conv1 / conv2: 3x3, pad 1.
  models/downsampling.py, Downsample2D (use_conv, padding 0): F.pad(x, (0, 1, 0, 1)) then 3x3 conv, stride 2, pad 0.
  models/upsampling.py, Upsample2D (use_conv): F.interpolate(x, scale_factor=2.0, mode="nearest") then 3x3 conv, pad 1.
  image_processor.py, VaeImageProcessor(vae_scale_factor, do_normalize=False)
    preprocess(PIL image): resize to (w // f * f, h // f * f) with PIL LANCZOS (resample="lanczos"), /255 -> fp32 NCHW in
    [0, 1]; no [-1, 1] mapping when do_normalize is False.
    postprocess(x, "pil"): no denormalisation when do_normalize is False; x.cpu().permute(0, 2, 3, 1).float().numpy(),
    then numpy_to_pil: (images * 255).round().astype("uint8").
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

# the aMUSEd 512 VQ-VAE configuration (vqvae/config.json of amused/amused-512)
AMUSED_CONFIG = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256, 256, 512, 768), layers_per_block=2,
                     latent_channels=64, num_vq_embeddings=8192, mid_block_add_attention=False, norm_num_groups=32)


def make_config(**kw):
    c = dict(AMUSED_CONFIG)
    c.update(kw)
    c["block_out_channels"] = tuple(c["block_out_channels"])
    return SimpleNamespace(**c)


def param_shapes(cfg) -> Dict[str, tuple]:
    """Names and shapes of every VQModel parameter under diffusers' registration names."""
    sh: Dict[str, tuple] = {}

    def conv(name, cout, cin, k):
        sh[name + ".weight"] = (cout, cin, k, k)
        sh[name + ".bias"] = (cout,)

    def lin(name, c):
        sh[name + ".weight"] = (c, c)
        sh[name + ".bias"] = (c,)

    def norm(name, c):
        sh[name + ".weight"] = (c,)
        sh[name + ".bias"] = (c,)

    def res(name, cin, cout):
        norm(name + ".norm1", cin)
        conv(name + ".conv1", cout, cin, 3)
        norm(name + ".norm2", cout)
        conv(name + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(name + ".conv_shortcut", cout, cin, 1)

    def mid(name, c):
        res(name + ".resnets.0", c, c)
        if cfg.mid_block_add_attention:
            norm(name + ".attentions.0.group_norm", c)
            for n in ("to_q", "to_k", "to_v", "to_out.0"):
                lin(name + ".attentions.0." + n, c)
        res(name + ".resnets.1", c, c)

    boc, L, lat, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.latent_channels, cfg.layers_per_block
    conv("encoder.conv_in", boc[0], cfg.in_channels, 3)
    cin = boc[0]
    for i in range(L):
        for j in range(lpb):
            res(f"encoder.down_blocks.{i}.resnets.{j}", cin if j == 0 else boc[i], boc[i])
        cin = boc[i]
        if i != L - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", boc[i], boc[i], 3)
    mid("encoder.mid_block", boc[-1])
    norm("encoder.conv_norm_out", boc[-1])
    conv("encoder.conv_out", lat, boc[-1], 3)
    conv("quant_conv", lat, lat, 1)
    sh["quantize.embedding.weight"] = (cfg.num_vq_embeddings, lat)
    conv("post_quant_conv", lat, lat, 1)
    conv("decoder.conv_in", boc[-1], lat, 3)
    mid("decoder.mid_block", boc[-1])
    rev = tuple(reversed(boc))
    cin = rev[0]
    for i in range(L):
        for j in range(lpb + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else rev[i], rev[i])
        cin = rev[i]
        if i != L - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", rev[i], rev[i], 3)
    norm("decoder.conv_norm_out", boc[0])
    conv("decoder.conv_out", cfg.out_channels, boc[0], 3)
    return sh


def make_weights(cfg, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights (fp32), fan-in scaled like oracle/magvit.py so activations stay O(1). The codebook is
    N(0, 1) rows: the encoder's latents have the same O(1) scale, so nearest-code search has real competition."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in param_shapes(cfg).items():
        if name == "quantize.embedding.weight":
            sd[name] = torch.randn(shape, generator=g)
        elif name.endswith(".weight") and len(shape) in (2, 4):
            fan_in = int(np.prod(shape[1:]))
            sd[name] = torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5
        elif len(shape) == 1 and "norm" in name and name.endswith(".weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            sd[name] = 0.05 * torch.randn(shape, generator=g)
    return sd


def _gn(x, w, name):
    return F.group_norm(x, 32, w[name + ".weight"], w[name + ".bias"], eps=1e-6)


def _conv(x, w, name, padding, stride=1):
    return F.conv2d(x, w[name + ".weight"], w[name + ".bias"], stride=stride, padding=padding)


def _res(x, w, name):
    h = _conv(F.silu(_gn(x, w, name + ".norm1")), w, name + ".conv1", 1)
    h = _conv(F.silu(_gn(h, w, name + ".norm2")), w, name + ".conv2", 1)
    if name + ".conv_shortcut.weight" in w:
        x = _conv(x, w, name + ".conv_shortcut", 0)
    return x + h


def _attn(x, w, name):
    b, c, h, wd = x.shape
    hs = _gn(x.view(b, c, h * wd), w, name + ".group_norm").transpose(1, 2)            # [B, hw, C]
    q, k, v = (F.linear(hs, w[f"{name}.{n}.weight"], w[f"{name}.{n}.bias"]) for n in ("to_q", "to_k", "to_v"))
    p = torch.softmax(torch.bmm(q, k.transpose(1, 2)) * c ** -0.5, dim=-1)
    o = F.linear(torch.bmm(p, v), w[name + ".to_out.0.weight"], w[name + ".to_out.0.bias"])
    return o.transpose(1, 2).reshape(b, c, h, wd) + x


def _mid(x, w, name, cfg):
    x = _res(x, w, name + ".resnets.0")
    if cfg.mid_block_add_attention:
        x = _attn(x, w, name + ".attentions.0")
    return _res(x, w, name + ".resnets.1")


@torch.no_grad()
def encode(x: torch.Tensor, w, cfg) -> torch.Tensor:
    """VQModel.encode(x).latents: pixels [B, 3, H, W] -> [B, latent_channels, H / 2^(L-1), W / 2^(L-1)]."""
    L = len(cfg.block_out_channels)
    h = _conv(x, w, "encoder.conv_in", 1)
    for i in range(L):
        for j in range(cfg.layers_per_block):
            h = _res(h, w, f"encoder.down_blocks.{i}.resnets.{j}")
        if i != L - 1:
            h = _conv(F.pad(h, (0, 1, 0, 1)), w, f"encoder.down_blocks.{i}.downsamplers.0.conv", 0, stride=2)
    h = _mid(h, w, "encoder.mid_block", cfg)
    h = _conv(F.silu(_gn(h, w, "encoder.conv_norm_out")), w, "encoder.conv_out", 1)
    return _conv(h, w, "quant_conv", 0)


@torch.no_grad()
def quantize(z: torch.Tensor, w):
    """VectorQuantizer.forward: (z_q NCHW with the straight-through form z + (z_q - z), flat indices in (b, y, x) order)."""
    emb = w["quantize.embedding.weight"]
    zf = z.permute(0, 2, 3, 1).contiguous()
    idx = torch.argmin(torch.cdist(zf.view(-1, emb.shape[1]), emb), dim=1)
    zq = emb[idx].view(zf.shape)
    zq = zf + (zq - zf)
    return zq.permute(0, 3, 1, 2).contiguous(), idx


def get_codebook_entry(indices: torch.Tensor, w, shape) -> torch.Tensor:
    """VectorQuantizer.get_codebook_entry(indices, shape=(B, h, w, C)) -> NCHW."""
    return w["quantize.embedding.weight"][indices].view(shape).permute(0, 3, 1, 2).contiguous()


@torch.no_grad()
def decode_latents(quant: torch.Tensor, w, cfg) -> torch.Tensor:
    """post_quant_conv + Decoder (norm_type 'group')."""
    L = len(cfg.block_out_channels)
    h = _conv(_conv(quant, w, "post_quant_conv", 0), w, "decoder.conv_in", 1)
    h = _mid(h, w, "decoder.mid_block", cfg)
    for i in range(L):
        for j in range(cfg.layers_per_block + 1):
            h = _res(h, w, f"decoder.up_blocks.{i}.resnets.{j}")
        if i != L - 1:
            h = _conv(F.interpolate(h, scale_factor=2.0, mode="nearest"), w, f"decoder.up_blocks.{i}.upsamplers.0.conv", 1)
    return _conv(F.silu(_gn(h, w, "decoder.conv_norm_out")), w, "decoder.conv_out", 1)


@torch.no_grad()
def decode(h: torch.Tensor, w, cfg, force_not_quantize=False, shape=None, lookup_from_codebook=True) -> torch.Tensor:
    """VQModel.decode(h, force_not_quantize, shape).sample."""
    if not force_not_quantize:
        quant = quantize(h, w)[0]
    elif lookup_from_codebook:
        quant = get_codebook_entry(h, w, shape)
    else:
        quant = h
    return decode_latents(quant, w, cfg)


# ---- VaeImageProcessor(vae_scale_factor, do_normalize=False) -------------------------------------------------------
def preprocess(img: Image.Image, vae_scale_factor: int) -> torch.Tensor:
    wd, ht = img.size
    wd, ht = (x - x % vae_scale_factor for x in (wd, ht))
    img = img.resize((wd, ht), resample=Image.LANCZOS)
    arr = np.array(img.convert("RGB")).astype(np.float32) / 255.0
    return torch.from_numpy(arr[None]).permute(0, 3, 1, 2).contiguous()


def postprocess(x: torch.Tensor):
    arr = x.detach().cpu().permute(0, 2, 3, 1).float().numpy()
    arr = (arr * 255).round().astype("uint8")
    return [Image.fromarray(a) for a in arr]


class VaeImageProcessor:
    """The subset of diffusers.image_processor.VaeImageProcessor that the reference glue calls."""

    def __init__(self, vae_scale_factor: int = 8, do_normalize: bool = True, **_):
        assert not do_normalize, "only do_normalize=False is restated"
        self.vae_scale_factor = vae_scale_factor

    def preprocess(self, image, *_, **__):
        return preprocess(image, self.vae_scale_factor)

    def postprocess(self, image, output_type="pil", **_):
        assert output_type == "pil"
        return postprocess(image)


class OracleVQModel:
    """diffusers.VQModel stand-in over the functional forward above (CPU, fp32): what the reference glue is run against."""

    def __init__(self, cfg, w):
        self.cfg, self.w = cfg, w
        self.config = SimpleNamespace(block_out_channels=cfg.block_out_channels, latent_channels=cfg.latent_channels,
                                      lookup_from_codebook=True, num_vq_embeddings=cfg.num_vq_embeddings)
        self.device = torch.device("cpu")

    def to(self, *_a, **_k):
        return self

    def encode(self, x):
        return SimpleNamespace(latents=encode(x, self.w, self.cfg))

    def quantize(self, z):
        zq, idx = quantize(z, self.w)
        return zq, None, (None, None, idx)

    def decode(self, h, force_not_quantize=False, return_dict=True, shape=None):
        return SimpleNamespace(sample=decode(h, self.w, self.cfg, force_not_quantize, shape))
