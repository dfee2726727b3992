"""Drop-in for the subset of `diffusers.VQModel` that variant A calls (the aMUSEd VQ-VAE; MMaDA-Parallel-A/utils/
image_utils.py: decode :13-75, encode :159-173 and :176-285), on the native context of csrc/vq_decoder.cu.

    VQModel(**config, max_batch=1, max_latent_cells=1024, device="cuda:0")
    VQModel.from_pretrained(path, subfolder="vqvae")     local directory: config.json + diffusion_pytorch_model.safetensors
    .encode(x).latents                                   Encoder + quant_conv, one C call
    .quantize(latents) -> (z_q, None, (None, None, indices[B*h*w]))   nearest code (exact fp32 argmin, csrc/vq_codebook.cu)
    .decode(h, force_not_quantize=False, shape=None).sample           diffusers' three branches, one C call

Numerics: convolutions and the mid-block attention run with TF32 products and fp32 accumulation (what cuDNN does for the
fp32 module on a GPU with TF32 allowed); GroupNorm statistics in fp64; the nearest-code search in exact fp32. z_q is the
chosen codebook row itself, where diffusers returns the straight-through z + (z_q - z), which equals it up to rounding.
Supported configurations: DownEncoderBlock2D / UpDecoderBlock2D blocks, norm_type "group" with 32 groups, SiLU, channel
counts that are multiples of 32, vq_embed_dim == latent_channels, no remap. Anything else raises ValueError.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import warnings
from types import SimpleNamespace
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import check, lib, ptr, stream_ptr

# diffusers renamed the attention parameters of the VAE mid-block; checkpoints saved before that use the old names
_DEPRECATED_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}

_KNOWN = {"in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels", "layers_per_block",
          "act_fn", "latent_channels", "sample_size", "num_vq_embeddings", "norm_num_groups", "vq_embed_dim",
          "scaling_factor", "norm_type", "mid_block_add_attention", "lookup_from_codebook", "force_upcast", "remap"}


class VQModelConfig(dict):
    """The model's configuration with attribute access (like diffusers' FrozenDict)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None


def validate_config(cfg: dict) -> None:
    """Raises ValueError for the configurations the native context does not implement."""
    boc = tuple(cfg["block_out_channels"])
    if not 1 <= len(boc) <= 8:
        raise ValueError(f"VQModel: {len(boc)} levels (block_out_channels) outside [1, 8]")
    if any(c <= 0 or c % 32 for c in boc):
        raise ValueError(f"VQModel: block_out_channels {boc} must be positive multiples of 32")
    if tuple(cfg["down_block_types"]) != ("DownEncoderBlock2D",) * len(boc):
        raise ValueError(f"VQModel: down_block_types {cfg['down_block_types']} (only DownEncoderBlock2D, one per level)")
    if tuple(cfg["up_block_types"]) != ("UpDecoderBlock2D",) * len(boc):
        raise ValueError(f"VQModel: up_block_types {cfg['up_block_types']} (only UpDecoderBlock2D, one per level)")
    if cfg["norm_type"] != "group":
        raise ValueError(f"VQModel: norm_type={cfg['norm_type']!r} (only 'group')")
    if cfg["act_fn"] != "silu":
        raise ValueError(f"VQModel: act_fn={cfg['act_fn']!r} (only 'silu')")
    if cfg["norm_num_groups"] != 32:
        raise ValueError(f"VQModel: norm_num_groups={cfg['norm_num_groups']} (only 32)")
    if cfg.get("remap") is not None:
        raise ValueError("VQModel: remap is not supported")
    if cfg["vq_embed_dim"] not in (None, cfg["latent_channels"]):
        raise ValueError(f"VQModel: vq_embed_dim={cfg['vq_embed_dim']} != latent_channels={cfg['latent_channels']}")
    if not 1 <= cfg["latent_channels"] <= 256:
        raise ValueError(f"VQModel: latent_channels={cfg['latent_channels']} outside [1, 256]")
    if not (1 <= cfg["in_channels"] <= 32 and 1 <= cfg["out_channels"] <= 32):
        raise ValueError("VQModel: in_channels / out_channels outside [1, 32]")
    if not 1 <= cfg["layers_per_block"] <= 16:
        raise ValueError(f"VQModel: layers_per_block={cfg['layers_per_block']} outside [1, 16]")
    if cfg["num_vq_embeddings"] < 1:
        raise ValueError(f"VQModel: num_vq_embeddings={cfg['num_vq_embeddings']}")


class VQModel:
    def __init__(self, in_channels: int = 3, out_channels: int = 3, down_block_types: Sequence[str] = ("DownEncoderBlock2D",),
                 up_block_types: Sequence[str] = ("UpDecoderBlock2D",), block_out_channels: Sequence[int] = (64,),
                 layers_per_block: int = 1, act_fn: str = "silu", latent_channels: int = 3, sample_size: int = 32,
                 num_vq_embeddings: int = 256, norm_num_groups: int = 32, vq_embed_dim: Optional[int] = None,
                 scaling_factor: float = 0.18215, norm_type: str = "group", mid_block_add_attention: bool = True,
                 lookup_from_codebook: bool = False, force_upcast: bool = False, remap=None, *, max_batch: int = 1,
                 max_latent_cells: int = 1024, device="cuda:0", **extra):
        # diffusers' defaults; keys of a config.json this class does not know are ignored (with a warning) like diffusers does
        unknown = sorted(k for k in extra if not k.startswith("_"))
        if unknown:
            warnings.warn(f"VQModel: ignoring config keys {unknown}")
        cfg = dict(in_channels=in_channels, out_channels=out_channels, down_block_types=tuple(down_block_types),
                   up_block_types=tuple(up_block_types), block_out_channels=tuple(block_out_channels),
                   layers_per_block=layers_per_block, act_fn=act_fn, latent_channels=latent_channels, sample_size=sample_size,
                   num_vq_embeddings=num_vq_embeddings, norm_num_groups=norm_num_groups, vq_embed_dim=vq_embed_dim,
                   scaling_factor=scaling_factor, norm_type=norm_type, mid_block_add_attention=bool(mid_block_add_attention),
                   lookup_from_codebook=bool(lookup_from_codebook), force_upcast=force_upcast, remap=remap)
        validate_config(cfg)
        if max_batch < 1 or max_latent_cells < 1:
            raise ValueError("VQModel: max_batch and max_latent_cells must be >= 1")
        self.config = VQModelConfig(cfg)
        if not torch.cuda.is_available():
            raise _lib.MmdpError("mmada_parallel_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.max_batch, self.max_latent_cells = max_batch, max_latent_cells
        self.scale = 2 ** (len(block_out_channels) - 1)
        c = _lib.VqModelConfig()
        c.in_channels, c.out_channels, c.n_levels = in_channels, out_channels, len(block_out_channels)
        for i, ch in enumerate(block_out_channels):
            c.block_out_channels[i] = ch
        c.layers_per_block, c.latent_channels, c.num_vq_embeddings = layers_per_block, latent_channels, num_vq_embeddings
        c.mid_block_add_attention = int(bool(mid_block_add_attention))
        c.max_batch, c.max_latent_cells = max_batch, max_latent_cells
        h = C.c_void_p()
        check(lib.mmdp_vqmodel_create(C.byref(c), C.byref(h)))
        self._h = h
        # device copy of the codebook for the nearest-code search (the context holds its own for the decode gather)
        self._codebook = torch.zeros((num_vq_embeddings, latent_channels), dtype=torch.float32, device=self.device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            lib.mmdp_vqdec_destroy(h)
            self._h = None

    # ---- construction / loading ---------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = "vqvae", *, max_batch: int = 1, max_latent_cells: int = 1024,
                        device="cuda:0", **_ignored) -> "VQModel":
        """Loads a LOCAL diffusers model directory (path[/subfolder]/config.json + diffusion_pytorch_model.safetensors).
        Hub ids are not resolved: there is no download."""
        root = os.path.join(path, subfolder) if subfolder else path
        cfg_path = os.path.join(root, "config.json")
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(f"VQModel.from_pretrained: {cfg_path} not found (a local directory is required)")
        with open(cfg_path) as f:
            cfg = json.load(f)
        from safetensors.torch import load_file
        st = os.path.join(root, "diffusion_pytorch_model.safetensors")
        if not os.path.isfile(st):
            raise FileNotFoundError(f"VQModel.from_pretrained: {st} not found")
        m = cls(**cfg, max_batch=max_batch, max_latent_cells=max_latent_cells, device=device)
        m.load_state_dict(load_file(st), strict=True)
        return m

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        unexpected = []
        for k, v in state_dict.items():
            parts = k.split(".")
            if len(parts) >= 2 and parts[-2] in _DEPRECATED_ATTN and ".attentions." in k:
                k_new = ".".join(parts[:-2] + [_DEPRECATED_ATTN[parts[-2]], parts[-1]])
            else:
                k_new = k
            t = v.detach().to(torch.float32).contiguous()
            if lib.mmdp_vqdec_set_weight(self._h, k_new.encode(), t.data_ptr(), t.numel(), stream_ptr()) != 0:
                unexpected.append(k)
            elif k_new == "quantize.embedding.weight":
                self._codebook.copy_(t.view(self._codebook.shape))
        torch.cuda.synchronize(self.device)
        buf = C.create_string_buffer(4096)
        n_missing = lib.mmdp_vqdec_missing(self._h, buf, 4096)
        missing = buf.value.decode().split()
        if strict and (n_missing or unexpected):
            raise RuntimeError(f"VQModel.load_state_dict: {n_missing} missing keys ({' '.join(missing[:8])}), "
                               f"unexpected keys {unexpected[:8]}")
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def eval(self):
        return self

    def to(self, *args, **kwargs):
        for a in list(args) + [kwargs.get("device")]:
            if isinstance(a, (str, torch.device)) and not isinstance(a, torch.dtype):
                d = torch.device(a)
                if d.type != "cuda" or (d.index is not None and d.index != self.device.index):
                    raise ValueError(f"VQModel lives on {self.device}; it cannot move to {d}")
        return self

    @property
    def dtype(self):
        return torch.float32

    # ---- forward ------------------------------------------------------------------------------------------------
    def _batch_check(self, b: int, h: int, w: int):
        if b < 1 or b > self.max_batch or h * w > self.max_latent_cells:
            raise ValueError(f"VQModel: batch {b}, latent grid {h}x{w} exceeds the context (max_batch={self.max_batch}, "
                             f"max_latent_cells={self.max_latent_cells})")

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        x = x.to(device=self.device, dtype=torch.float32).contiguous()
        if x.dim() != 4 or x.shape[1] != self.config.in_channels:
            raise ValueError(f"VQModel.encode: expected [B, {self.config.in_channels}, H, W], got {tuple(x.shape)}")
        b, _, hh, ww = x.shape
        if hh % self.scale or ww % self.scale or hh == 0 or ww == 0:
            raise ValueError(f"VQModel.encode: {hh}x{ww} pixels are not multiples of {self.scale}")
        self._batch_check(b, hh // self.scale, ww // self.scale)
        lat = torch.empty((b, self.config.latent_channels, hh // self.scale, ww // self.scale), dtype=torch.float32,
                          device=self.device)
        check(lib.mmdp_vqmodel_encode(self._h, ptr(x), b, hh, ww, ptr(lat), stream_ptr()))
        return SimpleNamespace(latents=lat) if return_dict else (lat,)

    @torch.no_grad()
    def quantize(self, z: torch.Tensor):
        """VectorQuantizer.forward: (z_q [B, C, h, w], None, (None, None, indices [B*h*w] in (b, y, x) order))."""
        z = z.to(device=self.device, dtype=torch.float32).contiguous()
        if z.dim() != 4 or z.shape[1] != self.config.latent_channels:
            raise ValueError(f"VQModel.quantize: expected [B, {self.config.latent_channels}, h, w], got {tuple(z.shape)}")
        b, c, h, w = z.shape
        ids = torch.empty(b * h * w, dtype=torch.int64, device=self.device)
        zq = torch.empty_like(z)
        check(lib.mmdp_vq_nearest(ptr(z), ptr(self._codebook), b, c, h, w, self.config.num_vq_embeddings, ptr(ids), ptr(zq),
                                  stream_ptr()))
        return zq, None, (None, None, ids)

    @torch.no_grad()
    def decode(self, h: torch.Tensor, force_not_quantize: bool = False, return_dict: bool = True, shape=None):
        lat_c = self.config.latent_channels
        if not force_not_quantize or not self.config.lookup_from_codebook:
            quant = self.quantize(h)[0] if not force_not_quantize else h.to(device=self.device, dtype=torch.float32).contiguous()
            if quant.dim() != 4 or quant.shape[1] != lat_c:
                raise ValueError(f"VQModel.decode: expected latents [B, {lat_c}, h, w], got {tuple(quant.shape)}")
            b, _, hh, ww = quant.shape
            ids = None
        else:
            ids = h.to(device=self.device, dtype=torch.int64).contiguous()
            if shape is not None:
                b, hh, ww, c = shape
                if c != lat_c:
                    raise ValueError(f"VQModel.decode: shape {tuple(shape)} has {c} channels, the codebook {lat_c}")
            elif ids.dim() == 3:
                b, hh, ww = ids.shape
            else:
                raise ValueError("VQModel.decode: codebook lookup needs shape=(B, h, w, C) or ids [B, h, w]")
            if ids.numel() != b * hh * ww:
                raise ValueError(f"VQModel.decode: {ids.numel()} ids do not fill shape {(b, hh, ww)}")
            quant = None
        self._batch_check(b, hh, ww)
        out = torch.empty((b, self.config.out_channels, hh * self.scale, ww * self.scale), dtype=torch.float32, device=self.device)
        check(lib.mmdp_vqmodel_decode(self._h, ptr(ids), ptr(quant), b, hh, ww, ptr(out), stream_ptr()))
        if ids is not None:
            flags = C.c_int32()
            check(lib.mmdp_vqmodel_error_flags(self._h, C.byref(flags), stream_ptr()))
            if flags.value & 1:
                raise IndexError(f"VQModel.decode: a codebook index is outside [0, {self.config.num_vq_embeddings})")
        return SimpleNamespace(sample=out) if return_dict else (out,)
