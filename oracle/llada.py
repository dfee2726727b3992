"""ORACLE (test infrastructure, NOT product code): CPU restatement of the LLaDA backbone forward on the inference path.

Restates MMaDA-Parallel-A/model/modeling_llada.py (identical in M/models/modeling_llada.py for this path):
  RMSLayerNorm.forward :315-329, RotaryEmbedding :376-435, LLaDALlamaBlock.forward :906-972,
  LLaDAModel.forward :1201-1415 (embedding, blocks, ln_f, ff_out head). Dead work of the reference (attention-bias
  construction that SDPA never receives, :1306-1316 / :718-727) is not restated because it cannot change outputs.
Every nn.Linear / elementwise op runs in the weights' dtype (bf16) with torch-CPU kernels, so the bf16 rounding
points are the reference's. Pinned against the real reference in tests/test_oracle_golden.py.
Also holds the deterministic synthetic-weight generator shared by the golden-vector script and the GPU tests.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn.functional as F


def make_config(d_model=256, n_heads=2, n_layers=2, mlp_hidden_size=512, vocab_size=134656, rope_theta=500000.0,
                rms_norm_eps=1e-5, max_sequence_length=1024) -> SimpleNamespace:
    """Field names follow model/configuration_llada.py:129-384 (ModelConfig)."""
    return SimpleNamespace(d_model=d_model, n_heads=n_heads, n_kv_heads=None, n_layers=n_layers,
                           mlp_hidden_size=mlp_hidden_size, mlp_ratio=4, vocab_size=vocab_size,
                           embedding_size=vocab_size, rope_theta=rope_theta, rms_norm_eps=rms_norm_eps,
                           max_sequence_length=max_sequence_length, rope=True, rope_full_precision=True,
                           include_bias=False, weight_tying=False, alibi=False, scale_logits=False,
                           input_emb_norm=False, attention_layer_norm=False, include_qkv_bias=False)


def make_weights(cfg, seed: int = 0, std: float = 0.02, dtype=torch.bfloat16, device="cpu",
                 head_std: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic state dict with the HF names of the reference checkpoint (SURVEY.md §8b).
    Values come from a seeded CPU torch.Generator so the fixture script (here) and the GPU tests (on the box, same
    image / same torch build) materialise bit-identical tensors without shipping them."""
    g = torch.Generator().manual_seed(seed)
    d, ff, V = cfg.d_model, cfg.mlp_hidden_size, cfg.embedding_size or cfg.vocab_size

    def rnd(*shape, s=std):
        return (torch.randn(*shape, generator=g) * s).to(dtype).to(device)

    sd = {"model.transformer.wte.weight": rnd(V, d)}
    for i in range(cfg.n_layers):
        p = f"model.transformer.blocks.{i}."
        sd[p + "q_proj.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "k_proj.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "v_proj.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "attn_out.weight"] = rnd(d, d, s=d ** -0.5)
        sd[p + "ff_proj.weight"] = rnd(ff, d, s=d ** -0.5)
        sd[p + "up_proj.weight"] = rnd(ff, d, s=d ** -0.5)
        sd[p + "ff_out.weight"] = rnd(d, ff, s=ff ** -0.5)
        sd[p + "attn_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
        sd[p + "ff_norm.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
    sd["model.transformer.ln_f.weight"] = (1.0 + 0.1 * torch.randn(d, generator=g)).to(dtype).to(device)
    sd["model.transformer.ff_out.weight"] = rnd(V, d, s=head_std if head_std is not None else d ** -0.5)
    return sd


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """RMSLayerNorm.forward, modeling_llada.py:315-329."""
    og_dtype = x.dtype
    xf = x.to(torch.float32)
    variance = xf.pow(2).mean(-1, keepdim=True)
    xf = xf * torch.rsqrt(variance + eps)
    return weight * xf.to(og_dtype)


def rotary_tables(head_dim: int, theta: float, seq_len: int):
    """RotaryEmbedding.get_rotary_embedding, modeling_llada.py:376-400 -> pos_sin, pos_cos [1,1,T,head_dim] fp32."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float) / head_dim))
    seq = torch.arange(seq_len, dtype=torch.float)
    freqs = torch.einsum("i , j -> i j", seq, inv_freq)
    positions = torch.cat((freqs, freqs), dim=-1)
    return positions.sin()[None, None, :, :], positions.cos()[None, None, :, :]


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    B, nh, T, hs = x.size()
    x = x.view(B, nh, T, 2, hs // 2)
    x1, x2 = x.unbind(dim=-2)
    return torch.cat((-x2, x1), dim=-1)                                            # :402-406


def apply_rotary(pos_sin, pos_cos, t):
    return ((t * pos_cos) + (rotate_half(t) * pos_sin)).to(t.dtype)                # :408-409


def block_forward(x: torch.Tensor, w: Dict[str, torch.Tensor], prefix: str, cfg, pos_sin, pos_cos) -> torch.Tensor:
    """LLaDALlamaBlock.forward, modeling_llada.py:906-972 (+ attention :681-744, SDPA :672-679)."""
    B, T, C = x.shape
    nh = cfg.n_heads
    xn = rms_norm(x, w[prefix + "attn_norm.weight"], cfg.rms_norm_eps)
    q = F.linear(xn, w[prefix + "q_proj.weight"])
    k = F.linear(xn, w[prefix + "k_proj.weight"])
    v = F.linear(xn, w[prefix + "v_proj.weight"])
    q = q.view(B, T, nh, C // nh).transpose(1, 2)
    k = k.view(B, T, nh, C // nh).transpose(1, 2)
    v = v.view(B, T, nh, C // nh).transpose(1, 2)
    q_ = apply_rotary(pos_sin, pos_cos, q.float()).type_as(q)                       # rope_full_precision, :412-435
    k_ = apply_rotary(pos_sin, pos_cos, k.float()).type_as(k)
    att = F.scaled_dot_product_attention(q_, k_, v, attn_mask=None, dropout_p=0.0, is_causal=False)
    att = att.transpose(1, 2).contiguous().view(B, T, C)
    x = x + F.linear(att, w[prefix + "attn_out.weight"])                            # :744, :953
    og_x = x
    h = rms_norm(x, w[prefix + "ff_norm.weight"], cfg.rms_norm_eps)
    g, up = F.linear(h, w[prefix + "ff_proj.weight"]), F.linear(h, w[prefix + "up_proj.weight"])
    h = F.silu(g) * up                                                              # :962-967
    return og_x + F.linear(h, w[prefix + "ff_out.weight"])                          # :968-970


def forward_hidden(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg) -> torch.Tensor:
    """Embedding + all blocks + ln_f -> [B, T, d] (modeling_llada.py:1265, :1333-1364, :1392)."""
    B, T = ids.shape
    x = F.embedding(ids, w["model.transformer.wte.weight"])
    pos_sin, pos_cos = rotary_tables(cfg.d_model // cfg.n_heads, cfg.rope_theta, T)
    pos_sin, pos_cos = pos_sin.to(x.device), pos_cos.to(x.device)  # (tables are built on the CPU like the checker's)
    for i in range(cfg.n_layers):
        x = block_forward(x, w, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos)
    return rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)


def forward_logits(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg) -> torch.Tensor:
    """LLaDAModel.forward -> logits [B, T, V] in the weight dtype (modeling_llada.py:1402)."""
    return F.linear(forward_hidden(ids, w, cfg), w["model.transformer.ff_out.weight"])


class OracleModel:
    """Callable with the reference wrapper's contract: model(ids, infer=True, use_cache=False).logits."""

    def __init__(self, cfg, weights: Dict[str, torch.Tensor]):
        self.config, self.w = cfg, weights
        self.device = next(iter(weights.values())).device

    @torch.no_grad()
    def __call__(self, input_ids, infer=True, use_cache=False, **_):
        ids = input_ids if torch.is_tensor(input_ids) else torch.tensor(input_ids)
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        return SimpleNamespace(logits=forward_logits(ids.to(self.device), self.w, self.config))


class CachedOracleModel:
    """Restates the token-cache forward of the reference: LLaDAModelLM.forward(input_ids, use_cache=True, to_compute_mask=mask,
    cat=key) after model.caching(True) - modeling_llada.py:1244-1245 (ids restricted to the masked tokens), :929-940 (per-block
    k / v caches: stored whole without a mask, scattered at the masked positions with one), :715-716 + :412-435 (rotary with the
    masked tokens' own positions for q, all positions for the cached k), :1406-1413 (logit cache; the cache tensor is what is
    returned). Pinned against the real reference in oracle/make_golden_cache.py.
    `linear(x, name)` computes the block linear whose weight is the state-dict entry `name` (q/k/v_proj, attn_out, ff_proj,
    up_proj, ff_out of a block; not the LM head). Default: F.linear in the weights' dtype, the reference's linear;
    oracle.fp8.linear_hook gives the FP8 block linears. Runs on the device its weights live on."""

    def __init__(self, cfg, weights: Dict[str, torch.Tensor], linear=None):
        self.config, self.w = cfg, weights
        self.linear = linear if linear is not None else (lambda x, name: F.linear(x, weights[name]))
        self.k, self.v, self.logit = {}, {}, {}

    def empty_cache(self):
        self.k, self.v, self.logit = {}, {}, {}

    @torch.no_grad()
    def __call__(self, input_ids, to_compute_mask=None, cat=""):
        cfg, w = self.config, self.w
        ids = input_ids
        B, L = ids.shape
        if to_compute_mask is not None:
            assert B == 1, "the reference's rotary indexing (nonzero()[1] of the whole mask, :715) only works for batch 1"
            ids = ids[to_compute_mask].view(B, -1)                                              # :1244-1245
        x = F.embedding(ids, w["model.transformer.wte.weight"])
        nh, C = cfg.n_heads, cfg.d_model
        pos_sin, pos_cos = (t.to(x.device) for t in rotary_tables(C // nh, cfg.rope_theta, L))
        lin = self.linear
        for i in range(cfg.n_layers):
            p = f"model.transformer.blocks.{i}."
            T = x.shape[1]
            xn = rms_norm(x, w[p + "attn_norm.weight"], cfg.rms_norm_eps)
            q, k, v = (lin(xn, p + n + ".weight") for n in ("q_proj", "k_proj", "v_proj"))
            key = (i, cat)
            if key not in self.k:                                                               # :930-932
                self.k[key] = torch.zeros(B, L, C, dtype=x.dtype, device=x.device)
                self.v[key] = torch.zeros(B, L, C, dtype=x.dtype, device=x.device)
            if to_compute_mask is not None:                                                     # :933-937
                self.k[key][to_compute_mask] = k.reshape(-1, C)
                self.v[key][to_compute_mask] = v.reshape(-1, C)
                k, v = self.k[key], self.v[key]
            else:                                                                               # :938-940
                self.k[key], self.v[key] = k, v
            qh = q.view(B, T, nh, C // nh).transpose(1, 2)
            kh = k.view(B, L, nh, C // nh).transpose(1, 2)
            vh = v.view(B, L, nh, C // nh).transpose(1, 2)
            if to_compute_mask is not None:                                                     # :715-716 -> :424-429
                qidx = to_compute_mask.nonzero(as_tuple=True)[1]
                q_ = apply_rotary(pos_sin[:, :, qidx, :], pos_cos[:, :, qidx, :], qh.float()).type_as(qh)
            else:
                q_ = apply_rotary(pos_sin, pos_cos, qh.float()).type_as(qh)
            k_ = apply_rotary(pos_sin, pos_cos, kh.float()).type_as(kh)
            att = F.scaled_dot_product_attention(q_, k_, vh, attn_mask=None, dropout_p=0.0, is_causal=False)
            att = att.transpose(1, 2).contiguous().view(B, T, C)
            x = x + lin(att, p + "attn_out.weight")
            h = rms_norm(x, w[p + "ff_norm.weight"], cfg.rms_norm_eps)
            h = F.silu(lin(h, p + "ff_proj.weight")) * lin(h, p + "up_proj.weight")
            x = x + lin(h, p + "ff_out.weight")
        x = rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)
        logits = F.linear(x, w["model.transformer.ff_out.weight"])
        if cat not in self.logit:                                                               # :1406-1413
            self.logit[cat] = torch.zeros_like(logits)
        if to_compute_mask is not None:
            self.logit[cat][to_compute_mask] = logits.view(-1, logits.shape[-1])
            logits = self.logit[cat]
        else:
            self.logit[cat] = logits
        return SimpleNamespace(logits=logits)
