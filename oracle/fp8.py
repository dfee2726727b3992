"""ORACLE (test infrastructure, NOT product code): definition of the opt-in FP8 (e4m3) precision of the block linears.

The reference has no FP8; these functions ARE the contract the CUDA path (csrc/fp8.cu, include/mmdp.h) is pinned to:
  quantize_fp8   s = amax|x| / 448 per row group (fp32, IEEE division; 1 for an all-zero group), q = e4m3(x / s)
  linear_fp8     acc[m, n] = sw[n] * sum_g sa[g, m] * (sum_{k in g} qa[m, k] * qw[n, k]) in fp32, groups of 128 along K
  block_forward_fp8 / forward_logits_fp8 / linear_hook
                 oracle.llada's block, forward and token-cache forward (CachedOracleModel) with the four linears
                 (q/k/v_proj, attn_out, ff_proj/up_proj, ff_out) replaced by bf16(linear_fp8(quantised input, quantised weight)); weights use one scale per row (group = K),
                 activations 1 x 128 groups. Every other op and bf16 rounding point is oracle.llada's.
Runs on whatever device its inputs live on (the tests use the CPU, and torch on the GPU for the large shapes).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from . import llada

E4M3_MAX = 448.0
ACT_GROUP = 128
_LINEARS = ("q_proj", "k_proj", "v_proj", "attn_out", "ff_proj", "up_proj", "ff_out")


def quantize_fp8(x: torch.Tensor, group: int):
    """x bf16 [rows, K] -> (q float8_e4m3fn [rows, K], s fp32 [K // group, rows]) - the layout of mmdp_quantize_fp8."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2
    rows, K = x.shape
    assert group > 0 and K % group == 0
    xf = x.float().reshape(rows, K // group, group)
    amax = xf.abs().amax(dim=-1)
    s = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    # |x / s| <= 448 * (1 + 2^-8) here (s may be an fp32 subnormal); torch's cast is NaN only from 464 on
    q = (xf / s.unsqueeze(-1)).to(torch.float8_e4m3fn)
    assert not torch.isnan(q.float()).any(), "quantize_fp8: value outside the e4m3 range"
    return q.reshape(rows, K), s.t().contiguous()


def linear_fp8(qa: torch.Tensor, sa: torch.Tensor, qw: torch.Tensor, sw: torch.Tensor) -> torch.Tensor:
    """qa [M, K] e4m3, sa [K/128, M]; qw [N, K] e4m3, sw [N] -> fp32 [M, N]. Products of e4m3 values are exact in fp32."""
    M, K = qa.shape
    N = qw.shape[0]
    G = ACT_GROUP
    a = qa.float().reshape(M, K // G, G)
    w = qw.float().reshape(N, K // G, G)
    acc = torch.zeros(M, N, dtype=torch.float32, device=qa.device)
    for g in range(K // G):
        acc = acc + sa[g].unsqueeze(1) * (a[:, g] @ w[:, g].t())
    return acc * sw.unsqueeze(0)


def quantize_weights(w: Dict[str, torch.Tensor]) -> Dict[str, tuple]:
    """(q, s) per linear weight of the blocks, one scale per row; keyed by the state-dict name."""
    out = {}
    for k, v in w.items():
        if k.endswith(".weight") and k.split(".")[-2] in _LINEARS and ".blocks." in k:
            q, s = quantize_fp8(v, v.shape[1])
            out[k] = (q, s[0])
    return out


def _linear(x: torch.Tensor, qw_sw) -> torch.Tensor:
    shape = x.shape
    qa, sa = quantize_fp8(x.reshape(-1, shape[-1]), ACT_GROUP)
    y = linear_fp8(qa, sa, *qw_sw).to(torch.bfloat16)
    return y.reshape(*shape[:-1], y.shape[-1])


def linear_hook(wq: Dict[str, tuple]):
    """llada.CachedOracleModel's `linear` with the block linears in FP8 (wq = quantize_weights(w))."""
    return lambda x, name: _linear(x, wq[name])


def block_forward_fp8(x: torch.Tensor, w: Dict[str, torch.Tensor], wq: Dict[str, tuple], prefix: str, cfg, pos_sin, pos_cos):
    """llada.block_forward with the four linears in FP8 (wq = quantize_weights(w))."""
    B, T, C = x.shape
    nh = cfg.n_heads
    xn = llada.rms_norm(x, w[prefix + "attn_norm.weight"], cfg.rms_norm_eps)
    q = _linear(xn, wq[prefix + "q_proj.weight"])
    k = _linear(xn, wq[prefix + "k_proj.weight"])
    v = _linear(xn, wq[prefix + "v_proj.weight"])
    q = q.view(B, T, nh, C // nh).transpose(1, 2)
    k = k.view(B, T, nh, C // nh).transpose(1, 2)
    v = v.view(B, T, nh, C // nh).transpose(1, 2)
    q_ = llada.apply_rotary(pos_sin, pos_cos, q.float()).type_as(q)
    k_ = llada.apply_rotary(pos_sin, pos_cos, k.float()).type_as(k)
    att = F.scaled_dot_product_attention(q_, k_, v, attn_mask=None, dropout_p=0.0, is_causal=False)
    att = att.transpose(1, 2).contiguous().view(B, T, C)
    x = x + _linear(att, wq[prefix + "attn_out.weight"])
    og_x = x
    h = llada.rms_norm(x, w[prefix + "ff_norm.weight"], cfg.rms_norm_eps)
    g, up = _linear(h, wq[prefix + "ff_proj.weight"]), _linear(h, wq[prefix + "up_proj.weight"])
    h = F.silu(g) * up
    return og_x + _linear(h, wq[prefix + "ff_out.weight"])


def forward_logits_fp8(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg, wq: Dict[str, tuple] | None = None) -> torch.Tensor:
    """llada.forward_logits with FP8 block linears -> bf16 logits [B, T, V] (embedding, ln_f and the head stay bf16)."""
    wq = wq if wq is not None else quantize_weights(w)
    B, T = ids.shape
    x = F.embedding(ids, w["model.transformer.wte.weight"])
    pos_sin, pos_cos = llada.rotary_tables(cfg.d_model // cfg.n_heads, cfg.rope_theta, T)
    pos_sin, pos_cos = pos_sin.to(x.device), pos_cos.to(x.device)
    for i in range(cfg.n_layers):
        x = block_forward_fp8(x, w, wq, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos)
    x = llada.rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)
    return F.linear(x, w["model.transformer.ff_out.weight"])
