"""Drop-in for the decode side of MMaDA-Parallel-M/models/modeling_magvitv2.py: `MAGVITv2.decode_code`
(:429-433) = LFQuantizer.get_codebook_entry (:208-221) + VQGANDecoder.forward (:365-399), as one C call into the native
decoder context (TF32 wgmma implicit-GEMM convolutions, csrc/conv_tf32.cu + csrc/vq_decoder.cu).

Numerics: the reference module runs in fp32; on a GPU its convolutions go through cuDNN with TF32 allowed (PyTorch
default), which is the precision of this implementation (10-bit mantissa products, fp32 accumulation). Tolerance against
the fp32 CPU oracle is stated in tests/test_gpu_magvit.py.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import check, lib, ptr, stream_ptr


class VQGANDecoder:
    def __init__(self, ch: int = 128, ch_mult: Sequence[int] = (1, 1, 2, 2, 4), num_res_blocks: Sequence[int] = (4, 4, 3, 4, 3),
                 z_channels: int = 13, out_ch: int = 3, latent_hw=(32, 32), max_batch: int = 1, device: str = "cuda:0"):
        if not torch.cuda.is_available():
            raise _lib.MmdpError("mmada_parallel_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.cfg = SimpleNamespace(ch=ch, ch_mult=tuple(ch_mult), num_res_blocks=tuple(num_res_blocks), z_channels=z_channels,
                                   out_ch=out_ch, latent_hw=tuple(latent_hw), max_batch=max_batch)
        c = _lib.VqDecConfig()
        c.ch, c.n_levels, c.z_channels, c.out_ch, c.max_batch = ch, len(ch_mult), z_channels, out_ch, max_batch
        c.latent_h, c.latent_w = latent_hw
        for i, (m, n) in enumerate(zip(ch_mult, num_res_blocks)):
            c.ch_mult[i], c.num_res_blocks[i] = m, n
        h = C.c_void_p()
        check(lib.mmdp_vqdec_create(C.byref(c), C.byref(h)))
        self._h = h
        self.upscale = 2 ** (len(ch_mult) - 1)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            lib.mmdp_vqdec_destroy(h)
            self._h = None

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], prefix: str = "decoder.", strict: bool = True):
        """Accepts the reference module's names, with the 'decoder.' prefix (MAGVITv2 state dict) or without it."""
        unexpected = []
        for k, v in state_dict.items():
            if k.startswith("encoder.") or k.startswith("quantize."):
                continue
            name = k if k.startswith("decoder.") else prefix + k
            t = v.detach().to(torch.float32).contiguous()
            rc = lib.mmdp_vqdec_set_weight(self._h, name.encode(), t.data_ptr(), t.numel(), stream_ptr())
            if rc != 0:
                unexpected.append(k)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(512)
        missing = lib.mmdp_vqdec_missing(self._h, buf, 512)
        if strict and (missing or unexpected):
            raise KeyError(f"VQGANDecoder.load_state_dict: {missing} missing ({buf.value.decode()[:200]}), unexpected={unexpected[:6]}")
        return SimpleNamespace(missing_keys=buf.value.decode().split(), unexpected_keys=unexpected)

    def parameter_shapes(self) -> Dict[str, tuple]:
        """Names and shapes of the parameters this decoder expects (the reference module's registration names, prefix
        'decoder.'): lets callers build or validate a state dict without instantiating the reference nn.Module."""
        c = self.cfg
        sh: Dict[str, tuple] = {}

        def add(name, *shape):
            sh[name + ".weight"] = shape
            sh[name + ".bias"] = (shape[0],)

        def res(name, cin, cout):
            add(name + ".norm1", cin)
            add(name + ".conv1", cout, cin, 3, 3)
            add(name + ".norm2", cout)
            add(name + ".conv2", cout, cout, 3, 3)
            if cin != cout:
                add(name + ".nin_shortcut", cout, cin, 1, 1)

        width = c.ch * c.ch_mult[-1]
        add("decoder.conv_in", width, c.z_channels, 3, 3)
        res("decoder.mid.block_1", width, width)
        add("decoder.mid.attn_1.norm", width)
        for n in ("q", "k", "v", "proj_out"):
            add("decoder.mid.attn_1." + n, width, width, 1, 1)
        res("decoder.mid.block_2", width, width)
        for lvl in range(len(c.ch_mult) - 1, -1, -1):
            out_w = c.ch * c.ch_mult[lvl]
            for blk in range(c.num_res_blocks[lvl]):
                res(f"decoder.up.{lvl}.block.{blk}", width, out_w)
                width = out_w
            if lvl:
                add(f"decoder.up.{lvl}.upsample.conv", width, width, 3, 3)
        add("decoder.norm_out", width)
        add("decoder.conv_out", c.out_ch, width, 3, 3)
        add("decoder.post_quant_conv", c.z_channels, c.z_channels, 1, 1)
        return sh

    def decode_ids(self, ids: torch.Tensor, shape=None) -> torch.Tensor:
        ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        b, n = ids.shape
        h, w = shape if shape is not None else (int(n ** 0.5), int(n ** 0.5))
        if h * w != n:
            raise ValueError(f"decode_code: {n} indices do not form a {h}x{w} grid")
        out = torch.empty((b, self.cfg.out_ch, h * self.upscale, w * self.upscale), dtype=torch.float32, device=self.device)
        check(lib.mmdp_vqdec_decode(self._h, ptr(ids), b, h, w, ptr(out), stream_ptr()))
        return out


class VQGANEncoder:
    """Encoder half (modeling_magvitv2.py:62-169): pixels [B, 3, H, W] -> 13-channel pre-quantisation map; `encode_ids`
    returns the LFQ code indices (MAGVITv2.get_code, :423-427) in one C call."""

    def __init__(self, ch: int = 128, ch_mult: Sequence[int] = (1, 2, 2, 4, 4), num_res_blocks: Sequence[int] = (4, 3, 4, 3, 4),
                 z_channels: int = 13, in_ch: int = 3, latent_hw=(32, 32), max_batch: int = 1, device: str = "cuda:0"):
        if not torch.cuda.is_available():
            raise _lib.MmdpError("mmada_parallel_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        c = _lib.VqDecConfig()
        c.ch, c.n_levels, c.z_channels, c.out_ch, c.max_batch = ch, len(ch_mult), z_channels, in_ch, max_batch
        c.latent_h, c.latent_w = latent_hw
        for i, (m, n) in enumerate(zip(ch_mult, num_res_blocks)):
            c.ch_mult[i], c.num_res_blocks[i] = m, n
        h = C.c_void_p()
        check(lib.mmdp_vqenc_create(C.byref(c), C.byref(h)))
        self._h = h
        self.downscale = 2 ** (len(ch_mult) - 1)
        self.in_ch = in_ch

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            lib.mmdp_vqdec_destroy(h)
            self._h = None

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        unexpected = []
        for k, v in state_dict.items():
            if k.startswith("decoder.") or k.startswith("quantize."):
                continue
            name = k if k.startswith("encoder.") else "encoder." + k
            t = v.detach().to(torch.float32).contiguous()
            if lib.mmdp_vqdec_set_weight(self._h, name.encode(), t.data_ptr(), t.numel(), stream_ptr()) != 0:
                unexpected.append(k)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(512)
        missing = lib.mmdp_vqdec_missing(self._h, buf, 512)
        if strict and (missing or unexpected):
            raise KeyError(f"VQGANEncoder.load_state_dict: {missing} missing ({buf.value.decode()[:200]}), unexpected={unexpected[:6]}")
        return SimpleNamespace(missing_keys=buf.value.decode().split(), unexpected_keys=unexpected)

    def encode_ids(self, pixels: torch.Tensor) -> torch.Tensor:
        x = pixels.to(device=self.device, dtype=torch.float32).contiguous()
        b, c, hh, ww = x.shape
        if c != self.in_ch or hh % self.downscale or ww % self.downscale:
            raise ValueError(f"get_code: expected [B, {self.in_ch}, H, W] with H, W multiples of {self.downscale}")
        ids = torch.empty((b, (hh // self.downscale) * (ww // self.downscale)), dtype=torch.int64, device=self.device)
        check(lib.mmdp_vqenc_encode(self._h, ptr(x), b, hh, ww, ptr(ids), stream_ptr()))
        return ids


class MAGVITv2:
    """Inference-side mirror of the reference class: `decode_code(ids[B, N], shape=None) -> FloatTensor[B, 3, H, W]` and
    `get_code(pixels[B, 3, H, W]) -> LongTensor[B, N]`. The encoder context is created on first use (encoder weights in
    the state dict, or the first get_code call)."""

    def __init__(self, max_batch: int = 1, device: str = "cuda:0", encoder_kw: Optional[dict] = None, **decoder_kw):
        self.decoder = VQGANDecoder(max_batch=max_batch, device=device, **decoder_kw)
        self.device = self.decoder.device
        self._enc_kw = dict(max_batch=max_batch, device=device, latent_hw=self.decoder.cfg.latent_hw, **(encoder_kw or {}))
        self.encoder: Optional[VQGANEncoder] = None

    def load_state_dict(self, state_dict, strict: bool = True):
        res = None
        if any(k.startswith("decoder.") for k in state_dict) or not any(k.startswith("encoder.") for k in state_dict):
            res = self.decoder.load_state_dict(state_dict, strict=strict)
        if any(k.startswith("encoder.") for k in state_dict):
            if self.encoder is None:
                self.encoder = VQGANEncoder(**self._enc_kw)
            res = self.encoder.load_state_dict(state_dict, strict=strict)
        return res

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    @torch.no_grad()
    def decode_code(self, codebook_indices: torch.Tensor, shape=None) -> torch.Tensor:
        return self.decoder.decode_ids(codebook_indices, shape=shape)

    @torch.no_grad()
    def get_code(self, pixel_values: torch.Tensor) -> torch.Tensor:
        if self.encoder is None:
            raise _lib.MmdpError("MAGVITv2.get_code: encoder weights were not loaded (state dict had no 'encoder.*' entries)")
        return self.encoder.encode_ids(pixel_values)
