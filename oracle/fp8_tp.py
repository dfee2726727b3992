"""ORACLE (test infrastructure, NOT product code): the FP8 (e4m3) block linears under tensor parallelism over `tp` ranks.

The contract the tensor-parallel FP8 path (TensorParallelLLaDA(precision="fp8"), csrc/api.cu mmdp_tp_forward, DESIGN §3 "FP8
under tensor parallel") is pinned to:
  * weights are quantised WHOLE (oracle.fp8.quantize_weights: one scale per row over the full K), then sliced. Rank r holds
    the rows of its heads / its ff columns for the column-parallel linears (q/k/v_proj, ff_proj/up_proj), and its K-columns
    of the bytes plus the FULL row scales for the row-parallel ones (attn_out, ff_out): shard_fp8;
  * activations are quantised in 1 x 128 groups along K. d_attn = 128 * heads per rank and ff / tp are multiples of 128, so a
    rank's K-slice holds whole groups, the single-GPU context's groups;
  * a column-parallel output element is the single-GPU element (same quantised input row, same weight row, same scale);
  * a row-parallel linear is the sum over ranks, in fp32 and in rank order, of the partials
        partial_r[m, n] = sw[n] * sum_{g in rank r} sa[g][m] * sum_{k in g} qa[m, k] qw[n, k]
    (oracle.fp8.linear_fp8 on the rank's K-slice), then x = bf16(bf16(sum) + x) as in the bf16 tensor-parallel forward.
At tp = 1 this is oracle.fp8_gqa's block bit for bit. Every other op is oracle.llada_gqa's (grouped-query, multi-query and
the q/k/v bias included).
"""
from __future__ import annotations

from typing import Dict

import torch

from . import fp8, fp8_gqa, llada, llada_gqa

_ROW_PARALLEL = ("attn_out", "ff_out")


def shard_fp8(wq: Dict[str, tuple], cfg, rank: int, tp: int) -> Dict[str, tuple]:
    """Rank `rank`'s slices of the quantised block linears (wq = oracle.fp8.quantize_weights(w)): name -> (q, s) with the q rows
    of the rank's heads, the k / v rows of the kv heads its query heads read (tp divides Hkv: its own share; Hkv divides tp: the
    one kv head, replicated), the rows of its ff columns, and the K-columns of attn_out / ff_out with their full row scales."""
    H, Hkv = cfg.n_heads, llada_gqa.kv_heads(cfg)
    Hl = H // tp
    kv0, n_kv = (rank * (Hkv // tp), Hkv // tp) if Hkv % tp == 0 else (rank * Hkv // tp, 1)
    heads, kvs = slice(rank * Hl * 128, (rank + 1) * Hl * 128), slice(kv0 * 128, (kv0 + n_kv) * 128)
    out = {}
    for name, (q, s) in wq.items():
        kind = name.split(".")[-2]
        if kind == "q_proj":
            out[name] = (q[heads], s[heads])
        elif kind in ("k_proj", "v_proj"):
            out[name] = (q[kvs], s[kvs])
        elif kind in ("ff_proj", "up_proj"):
            f = q.shape[0] // tp
            out[name] = (q[rank * f:(rank + 1) * f], s[rank * f:(rank + 1) * f])
        else:  # attn_out: K = d_model (heads), ff_out: K = mlp_hidden
            k = q.shape[1] // tp
            out[name] = (q[:, rank * k:(rank + 1) * k], s)
    return out


def row_parallel_fp8(x: torch.Tensor, qw_sw, tp: int) -> torch.Tensor:
    """The row-parallel linear of x [..., K] over tp ranks: fp32 sum in rank order of the per-rank partials -> bf16."""
    shape = x.shape
    qa, sa = fp8.quantize_fp8(x.reshape(-1, shape[-1]), fp8.ACT_GROUP)
    qw, sw = qw_sw
    K = qa.shape[1]
    k, g = K // tp, K // tp // fp8.ACT_GROUP
    assert k % fp8.ACT_GROUP == 0, "a rank's K-slice must hold whole 1 x 128 groups"
    total = None
    for r in range(tp):
        part = fp8.linear_fp8(qa[:, r * k:(r + 1) * k], sa[r * g:(r + 1) * g], qw[:, r * k:(r + 1) * k], sw)
        total = part if total is None else total + part
    y = total.to(torch.bfloat16)
    return y.reshape(*shape[:-1], y.shape[-1])


def block_forward_tp_fp8(x: torch.Tensor, w: Dict[str, torch.Tensor], wq: Dict[str, tuple], prefix: str, cfg, pos_sin, pos_cos,
                         tp: int) -> torch.Tensor:
    """oracle.fp8_gqa.block_forward_fp8 with attn_out and ff_out as tp-rank row-parallel sums."""
    def linear(t, name, b):
        if name.split(".")[-2] in _ROW_PARALLEL:
            return row_parallel_fp8(t, wq[name], tp)
        return fp8_gqa._linear(t, wq[name], b)
    return llada_gqa.attention_block(x, w, prefix, cfg, pos_sin, pos_cos, linear)


def hidden_tp_fp8(ids: torch.Tensor, w: Dict[str, torch.Tensor], cfg, tp: int, wq: Dict[str, tuple] | None = None) -> torch.Tensor:
    """ln_f(x) after all blocks [B, T, d] (what the tensor-parallel forward leaves in every rank's xn)."""
    wq = wq if wq is not None else fp8.quantize_weights(w)
    x = torch.nn.functional.embedding(ids, w["model.transformer.wte.weight"])
    pos_sin, pos_cos = llada.rotary_tables(cfg.d_model // cfg.n_heads, cfg.rope_theta, ids.shape[1])
    pos_sin, pos_cos = pos_sin.to(x.device), pos_cos.to(x.device)
    for i in range(cfg.n_layers):
        x = block_forward_tp_fp8(x, w, wq, f"model.transformer.blocks.{i}.", cfg, pos_sin, pos_cos, tp)
    return llada.rms_norm(x, w["model.transformer.ln_f.weight"], cfg.rms_norm_eps)
