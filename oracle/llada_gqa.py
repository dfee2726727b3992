"""ORACLE (test infrastructure, NOT product code): oracle.llada's backbone forward for grouped-query / multi-query attention and
the q/k/v projection bias.

Restates MMaDA-Parallel-A/model/modeling_llada.py for configs oracle.llada does not cover:
  ModelConfig.effective_n_kv_heads (configuration_llada.py:366-384), k_proj / v_proj with effective_n_kv_heads * head_dim rows and
  q/k/v_proj with a bias under include_qkv_bias (:866-884), rotary on the kv heads, then repeat_interleave of k / v to n_heads
  before SDPA (:653-679, :700-716).
Every other op is oracle.llada's, so the bf16 rounding points are the reference's; for n_kv_heads == n_heads without a bias the
results equal oracle.llada's. Pinned against the real reference in oracle/make_golden_gqa.py (tests/golden/forward_gqa_tiny.pt).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import llada


def make_config(n_kv_heads=None, multi_query_attention=None, include_qkv_bias=False, **kw) -> SimpleNamespace:
    """oracle.llada.make_config plus the three attention-layout fields of ModelConfig."""
    cfg = llada.make_config(**kw)
    cfg.n_kv_heads, cfg.multi_query_attention, cfg.include_qkv_bias = n_kv_heads, multi_query_attention, include_qkv_bias
    return cfg


def kv_heads(cfg) -> int:
    """ModelConfig.effective_n_kv_heads, configuration_llada.py:366-384."""
    n_kv, mqa = getattr(cfg, "n_kv_heads", None), getattr(cfg, "multi_query_attention", None)
    if n_kv is None:
        return 1 if mqa is True else cfg.n_heads
    if mqa is None:
        return n_kv
    should = 1 if mqa else cfg.n_heads
    if n_kv != should:
        raise Exception("You can't set `multi_query_attention` and `n_kv_heads` at the same time.")
    return should


def make_weights(cfg, seed: int = 0, std: float = 0.02, dtype=torch.bfloat16, device="cpu",
                 head_std: Optional[float] = None, bias_std: float = 0.25) -> Dict[str, torch.Tensor]:
    """oracle.llada.make_weights with k_proj / v_proj of kv_heads(cfg) * head_dim rows (the same draws in the same order, so a
    multi-head config gives oracle.llada's tensors) and, with include_qkv_bias, seeded non-zero q/k/v biases drawn after every
    other tensor (the reference initialises them to zero)."""
    g = torch.Generator().manual_seed(seed)
    d, ff, V = cfg.d_model, cfg.mlp_hidden_size, cfg.embedding_size or cfg.vocab_size
    dkv = kv_heads(cfg) * (d // cfg.n_heads)

    def rnd(*shape, s=std):
        return (torch.randn(*shape, generator=g) * s).to(dtype).to(device)

    sd = {"model.transformer.wte.weight": rnd(V, d)}
    for i in range(cfg.n_layers):
        p = f"model.transformer.blocks.{i}."
        sd[p + "q_proj.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "k_proj.weight"] = rnd(dkv, d, s=d ** -0.5)
        sd[p + "v_proj.weight"] = rnd(dkv, d, s=d ** -0.5)
        sd[p + "attn_out.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "ff_proj.weight"] = rnd(ff, d, s=d ** -0.5)
        sd[p + "up_proj.weight"] = rnd(ff, d, s=d ** -0.5)
        sd[p + "ff_out.weight"] = rnd(d, ff, s=ff ** -0.5)
        sd[p + "attn_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
        sd[p + "ff_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
    sd["model.transformer.ln_f.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
    sd["model.transformer.ff_out.weight"] = rnd(V, d, s=head_std if head_std is not None else d ** -0.5)
    if getattr(cfg, "include_qkv_bias", False):
        for i in range(cfg.n_layers):
            p = f"model.transformer.blocks.{i}."
            for n in ("q_proj", "k_proj", "v_proj"):
                sd[p + n + ".bias"] = rnd(sd[p + n + ".weight"].shape[0], s=bias_std)
    return sd


def grouped_kv(k: torch.Tensor, v: torch.Tensor, nh: int):
    """k / v [B, n_kv, T, hs] -> [B, nh, T, hs]: kv head j serves query heads [j G, (j + 1) G) (modeling_llada.py:663-670)."""
    if k.size(1) == nh:
        return k, v
    return (k.repeat_interleave(nh // k.size(1), dim=1, output_size=nh),
            v.repeat_interleave(nh // v.size(1), dim=1, output_size=nh))


def attention_block(x: torch.Tensor, w: Dict[str, torch.Tensor], prefix: str, cfg, pos_sin, pos_cos, linear) -> torch.Tensor:
    """LLaDALlamaBlock.forward with kv_heads(cfg) kv heads and optional q/k/v biases; `linear(x, name, bias)` runs one block linear
    (bf16 F.linear here, oracle.fp8_gqa's e4m3 linear there)."""
    B, T, C = x.shape
    nh, nkv = cfg.n_heads, kv_heads(cfg)
    xn = llada.rms_norm(x, w[prefix + "attn_norm.weight"], cfg.rms_norm_eps)
    q = linear(xn, prefix + "q_proj.weight", w.get(prefix + "q_proj.bias"))
    k = linear(xn, prefix + "k_proj.weight", w.get(prefix + "k_proj.bias"))
    v = linear(xn, prefix + "v_proj.weight", w.get(prefix + "v_proj.bias"))
    q = q.view(B, T, nh, C // nh).transpose(1, 2)
    k = k.view(B, T, nkv, C // nh).transpose(1, 2)
    v = v.view(B, T, nkv, C // nh).transpose(1, 2)
    q_ = llada.apply_rotary(pos_sin, pos_cos, q.float()).type_as(q)                 # rope_full_precision, :412-435
    k_ = llada.apply_rotary(pos_sin, pos_cos, k.float()).type_as(k)
    k_, v = grouped_kv(k_, v, nh)
    att = F.scaled_dot_product_attention(q_, k_, v, attn_mask=None, dropout_p=0.0, is_causal=False)
    att = att.transpose(1, 2).contiguous().view(B, T, C)
    x = x + linear(att, prefix + "attn_out.weight", None)                            # :744, :953
    og_x = x
    h = llada.rms_norm(x, w[prefix + "ff_norm.weight"], cfg.rms_norm_eps)
    g, up = linear(h, prefix + "ff_proj.weight", None), linear(h, prefix + "up_proj.weight", None)
    h = F.silu(g) * up                                                              # :962-967
    return og_x + linear(h, prefix + "ff_out.weight", None)                         # :968-970


def block_forward(x: torch.Tensor, w: Dict[str, torch.Tensor], prefix: str, cfg, pos_sin, pos_cos) -> torch.Tensor:
    """oracle.llada.block_forward for grouped-query configs (nn.Linear with bias = F.linear(x, W, b))."""
    return attention_block(x, w, prefix, cfg, pos_sin, pos_cos, lambda t, name, b: F.linear(t, w[name], b))


def forward_logits(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg, block=block_forward) -> torch.Tensor:
    """LLaDAModel.forward -> logits [B, T, V] (embedding, blocks, ln_f, head: oracle.llada.forward_logits' sequence)."""
    B, T = ids.shape
    x = F.embedding(ids, w["model.transformer.wte.weight"])
    pos_sin, pos_cos = llada.rotary_tables(cfg.d_model // cfg.n_heads, cfg.rope_theta, T)
    pos_sin, pos_cos = pos_sin.to(x.device), pos_cos.to(x.device)
    for i in range(cfg.n_layers):
        x = block(x, w, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos)
    x = llada.rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)
    return F.linear(x, w["model.transformer.ff_out.weight"])


class OracleModel(llada.OracleModel):
    """oracle.llada.OracleModel for grouped-query configs."""

    @torch.no_grad()
    def __call__(self, input_ids, infer=True, use_cache=False, **_):
        ids = input_ids if torch.is_tensor(input_ids) else torch.tensor(input_ids)
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        return SimpleNamespace(logits=forward_logits(ids.to(self.device), self.w, self.config))
