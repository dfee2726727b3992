"""ORACLE (test infrastructure, NOT product code): oracle.fp8's FP8 (e4m3) block linears for grouped-query / multi-query attention
and the q/k/v bias (oracle.llada_gqa's block).

Each block linear is bf16(linear_fp8(quantised input, quantised weight) + bias): the bias (q/k/v_proj with include_qkv_bias)
joins the fp32 result before the one bf16 rounding, as in the CUDA path's QKV epilogue. Quantisation and the e4m3 product are
oracle.fp8's; every other op is oracle.llada_gqa's.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import fp8, llada_gqa


def _linear(x: torch.Tensor, qw_sw, bias: torch.Tensor | None) -> torch.Tensor:
    shape = x.shape
    qa, sa = fp8.quantize_fp8(x.reshape(-1, shape[-1]), fp8.ACT_GROUP)
    y = fp8.linear_fp8(qa, sa, *qw_sw)
    if bias is not None:
        y = y + bias.float()
    y = y.to(torch.bfloat16)
    return y.reshape(*shape[:-1], y.shape[-1])


def block_forward_fp8(x: torch.Tensor, w: Dict[str, torch.Tensor], wq: Dict[str, tuple], prefix: str, cfg, pos_sin, pos_cos):
    """oracle.llada_gqa.block_forward with the four linears in FP8 (wq = oracle.fp8.quantize_weights(w))."""
    return llada_gqa.attention_block(x, w, prefix, cfg, pos_sin, pos_cos, lambda t, name, b: _linear(t, wq[name], b))


def forward_logits_fp8(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg, wq: Dict[str, tuple] | None = None) -> torch.Tensor:
    """oracle.llada_gqa.forward_logits with FP8 block linears -> bf16 logits [B, T, V] (embedding, ln_f and the head stay bf16)."""
    wq = wq if wq is not None else fp8.quantize_weights(w)
    return llada_gqa.forward_logits(ids, w, cfg,
                                    block=lambda x, w_, p, c, s, co: block_forward_fp8(x, w_, wq, p, c, s, co))
