"""Host-side mirror of the reference model objects for the denoising hot path.

`LLaDAForMultiModalGeneration` keeps the call contract of the reference wrapper
(MMaDA-Parallel-A/model/modeling_xllmx_dimoo.py:41-72): ``model(input_ids, infer=True, use_cache=False).logits``
returns bf16 logits ``[B, L, V]`` on ``model.device``. Underneath, weights live in device buffers owned by the native
context (libmmdp.so, include/mmdp.h) and one forward is a single C call that launches the sm_90a kernels.

The same object also exposes ``forward_rows`` - the restricted LM head the generators use so the full ``[L, V]``
logits never hit HBM (only text rows x V and image rows x codebook columns are computed).
"""
from __future__ import annotations

import ctypes as C
import json
import os
from types import SimpleNamespace
from typing import Dict, Iterable, Optional, Tuple

import torch

from . import _lib
from ._lib import lib, check, ptr, stream_ptr


class ModelOutput(SimpleNamespace):
    """Stand-in for transformers' CausalLMOutputWithPast: only `.logits` is meaningful on the inference path."""


def rope_tables(head_dim: int, theta: float, seq_len: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos/sin tables [seq_len, head_dim/2], computed with the reference's exact op sequence on the CPU
    (RotaryEmbedding.get_rotary_embedding, modeling_llada.py:376-400). The reference table is cat(freqs, freqs),
    so its second half is a copy of the first; only the first half is stored."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float) / head_dim))
    seq = torch.arange(seq_len, dtype=torch.float)
    freqs = torch.einsum("i , j -> i j", seq, inv_freq)
    return freqs.cos().contiguous(), freqs.sin().contiguous()


_BLOCK_KEYS = ("q_proj", "k_proj", "v_proj", "attn_out", "ff_proj", "up_proj", "ff_out", "attn_norm", "ff_norm")


def check_supported_config(config, n_heads: int) -> None:
    """Features of the reference config this path does not implement must fail loudly, not silently differ (shared by the
    single-GPU and the tensor-parallel model)."""
    g = lambda k, dflt=None: getattr(config, k, dflt)
    if g("n_kv_heads") not in (None, n_heads):
        raise NotImplementedError("GQA/MQA (n_kv_heads != n_heads) is not on the MMaDA-Parallel hot path")
    for flag in ("alibi", "include_bias", "include_qkv_bias", "weight_tying", "scale_logits", "input_emb_norm",
                 "attention_layer_norm"):
        if g(flag, False):
            raise NotImplementedError(f"config.{flag}=True is not supported by the H100 hot path")
    if not g("rope", True) or not g("rope_full_precision", True):
        raise NotImplementedError("the hot path implements full-precision RoPE only")
    # the kernels implement LLaDALlamaBlock + SwiGLU(silu) + RMSLayerNorm only (modeling_llada.py:906-972, :315-329);
    # a config that asks for another block / activation / norm must not be computed as if it were this one
    for key, ok in (("block_type", ("llama",)), ("activation_type", ("silu", "swiglu")), ("layer_norm_type", ("rms",))):
        v = g(key, None)
        v = getattr(v, "value", v)  # the reference uses StrEnum members
        if v is not None and str(v).lower() not in ok:
            raise NotImplementedError(f"config.{key}={v!r} is not supported by the H100 hot path (needs one of {ok})")


class LLaDAForMultiModalGeneration:
    """H100-native drop-in for the reference's inference-time model object (variant A wrapper and, through
    `MMadaModelLM` in mmada.py, variant M)."""

    def __init__(self, config, max_seq_len: Optional[int] = None, max_batch: int = 3, device: str = "cuda:0"):
        if not torch.cuda.is_available():
            raise _lib.MmdpError("mmada_parallel_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.config = config
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        g = lambda k, dflt=None: getattr(config, k, dflt)
        self.d_model = int(g("d_model"))
        self.n_heads = int(g("n_heads"))
        self.n_layers = int(g("n_layers"))
        self.mlp_hidden = int(g("mlp_hidden_size") or g("mlp_ratio", 4) * self.d_model)
        self.vocab_rows = int(g("embedding_size") or g("vocab_size"))
        self.rms_eps = float(g("rms_norm_eps", 1e-5))
        self.rope_theta = float(g("rope_theta", 10000.0))
        self.max_seq_len = int(max_seq_len or g("max_sequence_length", 4096))
        self.max_batch = int(max_batch)
        check_supported_config(config, self.n_heads)
        cfg = _lib.ModelConfig(self.d_model, self.n_heads, self.n_layers, self.mlp_hidden, self.vocab_rows,
                               self.max_seq_len, self.max_batch, self.rms_eps)
        handle = C.c_void_p()
        check(lib.mmdp_model_create(C.byref(cfg), C.byref(handle)))
        self._h = handle
        cos, sin = rope_tables(self.d_model // self.n_heads, self.rope_theta, self.max_seq_len)
        check(lib.mmdp_model_set_rope(self._h, cos.data_ptr(), sin.data_ptr(), self.max_seq_len, stream_ptr()))
        torch.cuda.synchronize()  # host tables may be freed after this point
        self._loaded: set = set()

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            lib.mmdp_model_destroy(h)
            self._h = None

    # ------------------------------------------------------------------------------------------------------------
    # weights
    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _native_name(hf_name: str) -> Optional[str]:
        n = hf_name
        if n.startswith("model."):
            n = n[len("model."):]
        if n.startswith("transformer."):
            n = n[len("transformer."):]
        if n == "wte.weight":
            return "wte"
        if n == "ln_f.weight":
            return "ln_f"
        if n == "ff_out.weight":
            return "head"
        if n.startswith("blocks."):
            parts = n.split(".")
            if len(parts) == 4 and parts[3] == "weight" and parts[2] in _BLOCK_KEYS:
                return f"blocks.{parts[1]}.{parts[2]}"
        return None

    def set_weight(self, hf_name: str, tensor: torch.Tensor) -> bool:
        name = self._native_name(hf_name)
        if name is None:
            return False
        t = tensor.detach().to(torch.bfloat16).contiguous()
        rows, cols = (t.shape[0], t.shape[1]) if t.dim() == 2 else (t.shape[0], 1)
        check(lib.mmdp_model_set_weight(self._h, name.encode(), t.data_ptr(), rows, cols, stream_ptr()))
        if not t.is_cuda:
            torch.cuda.synchronize()  # the async copy reads host memory that `t` owns
        self._loaded.add(name)
        return True

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor] | Iterable, strict: bool = True):
        items = state_dict.items() if hasattr(state_dict, "items") else state_dict
        unexpected = [k for k, v in items if not self.set_weight(k, v)]
        torch.cuda.synchronize()
        expected = {"wte", "ln_f", "head"} | {f"blocks.{i}.{k}" for i in range(self.n_layers) for k in _BLOCK_KEYS}
        missing = sorted(expected - self._loaded)
        if strict and (missing or unexpected):
            raise KeyError(f"load_state_dict: missing={missing[:8]} unexpected={unexpected[:8]}")
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    @classmethod
    def from_reference_module(cls, ref_model, **kw) -> "LLaDAForMultiModalGeneration":
        """Build from an instantiated reference nn.Module (used by the parity tooling in this container)."""
        m = cls(ref_model.config, **kw)
        m.load_state_dict(ref_model.state_dict())
        return m

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=torch.bfloat16, device_map=None, max_batch: int = 3,
                        device: str = "cuda:0", **_) -> "LLaDAForMultiModalGeneration":
        """Loads a HF checkpoint directory (config.json + *.safetensors), mirroring the call at A/inference.py:83-85."""
        from safetensors import safe_open

        with open(os.path.join(path, "config.json")) as f:
            cfg = SimpleNamespace(**json.load(f))
        m = cls(cfg, max_batch=max_batch, device=device)
        files = sorted(f for f in os.listdir(path) if f.endswith(".safetensors"))
        if not files:
            raise FileNotFoundError(f"no *.safetensors under {path}")
        for fn in files:
            with safe_open(os.path.join(path, fn), framework="pt", device="cpu") as sf:
                for k in sf.keys():
                    m.set_weight(k, sf.get_tensor(k))
        m.load_state_dict({}, strict=True)
        return m

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def parameters(self):
        """The reference's generators probe the device with `next(model.parameters()).device` (image_generation_generator.py:54)."""
        yield torch.empty(0, dtype=torch.bfloat16, device=self.device)

    def caching(self, enable: bool = True) -> None:
        """Mirror of LLaDAModel.caching (modeling_llada.py:1417-1421): switches the token cache on / off and drops what it holds.
        With the cache on, `model(ids, infer=True, use_cache=True, to_compute_mask=mask, cat=key)` recomputes only the masked
        tokens against the cached keys / values (see `forward`). The reference's own generators switch it on but never pass a
        mask (generate_image :65-68, :127), which leaves every output unchanged - also true here."""
        self._caching = bool(enable)
        self._cache = {}

    def empty_cache(self) -> None:
        """Mirror of LLaDAModel.empty_cache (modeling_llada.py:1423-1426)."""
        self._cache = {}

    def _forward_cached(self, ids: torch.Tensor, to_compute_mask: Optional[torch.Tensor], cat: str) -> torch.Tensor:
        """Token-cache forward (modeling_llada.py:1244-1245, :929-940, :715-716, :1406-1413) on the native context: a call without a
        mask is a full forward that (re)fills the per-block key / value caches and the logit cache of `cat`; a call with
        `to_compute_mask [B, L]` embeds only the masked tokens, refreshes their keys / values inside the caches, attends from them
        to ALL cached keys, and scatters their logits into the logit cache. Returns the logit cache itself, like the reference
        (the tensor is updated in place by later calls)."""
        B, L = ids.shape
        Lpad = (L + 7) // 8 * 8
        ent = self._cache.get(cat)
        if ent is not None and ent["shape"] != (B, L):
            raise ValueError(f"token cache '{cat}' holds a {ent['shape']} sequence, got {(B, L)}; call empty_cache() first")
        if ent is None:
            if to_compute_mask is not None:
                raise ValueError(f"token cache '{cat}' is empty: run a full forward (to_compute_mask=None) before a partial one")
            ent = {"shape": (B, L),
                   "k": torch.empty((self.n_layers, B * L, self.d_model), dtype=torch.bfloat16, device=self.device),
                   "vt": torch.zeros((self.n_layers, B, self.n_heads, 128, Lpad), dtype=torch.bfloat16, device=self.device),
                   "logits": torch.empty((B, L, self.vocab_rows), dtype=torch.bfloat16, device=self.device)}
            self._cache[cat] = ent
        if to_compute_mask is None:
            check(lib.mmdp_model_forward_cached(self._h, ptr(ids), B, L, L, None, ptr(ent["k"]), ptr(ent["vt"]), ptr(ent["logits"]),
                                                stream_ptr()))
            return ent["logits"]
        mask = to_compute_mask.to(device=self.device, dtype=torch.bool)
        if B != 1:
            raise ValueError("a partial forward is single-sample: the reference indexes the rotary table with nonzero()[1] of the "
                             "whole [B, L] mask (modeling_llada.py:715) and raises for B > 1")
        if tuple(mask.shape) != (B, L):
            raise ValueError("to_compute_mask must be a bool tensor of the shape of input_ids")
        counts = mask.sum(dim=1)
        tq = int(counts[0])
        if tq == 0 or bool((counts != tq).any()):
            raise ValueError("to_compute_mask must select the same non-zero number of tokens in every batch row "
                             "(the reference reshapes the selection with .view(batch, -1))")
        pos = mask.nonzero(as_tuple=False)[:, 1].to(torch.int32).contiguous()                       # increasing within each batch row
        ids_c = ids[mask].contiguous()                                                               # :1244-1245
        part = torch.empty((B * tq, self.vocab_rows), dtype=torch.bfloat16, device=self.device)
        check(lib.mmdp_model_forward_cached(self._h, ptr(ids_c), B, L, tq, ptr(pos), ptr(ent["k"]), ptr(ent["vt"]), ptr(part), stream_ptr()))
        ent["logits"][mask] = part                                                                   # :1409-1411
        return ent["logits"]

    supports_row_window = True   # forward_rows(row_window=...): generators/parallel_generator.py

    def raise_device_errors(self) -> None:
        """Reads and clears the sticky device-side error flags of the forwards issued so far (synchronises the stream).
        The kernels never read out of bounds; they flag what torch would have raised for."""
        flags = C.c_int32(0)
        check(lib.mmdp_model_error_flags(self._h, C.byref(flags), stream_ptr()))
        if flags.value & 1:
            raise IndexError("index out of range in self (a token id is outside [0, vocab_size))")
        if flags.value & 2:
            raise IndexError("a logits row index is outside [0, batch * seq_len)")
        if flags.value & 4:
            raise IndexError("a logits row index is outside the row window given to forward_rows")

    # ------------------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------------------
    def _ids_device(self, input_ids) -> torch.Tensor:
        if not torch.is_tensor(input_ids):
            # the reference wrapper accepts ragged python lists and right-pads with 0 (modeling_xllmx_dimoo.py:56-59)
            mx = max(len(r) for r in input_ids)
            input_ids = torch.tensor([list(r) + [0] * (mx - len(r)) for r in input_ids], dtype=torch.int64)
        ids = input_ids.to(device=self.device, dtype=torch.int64)
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        return ids.contiguous()

    def forward(self, input_ids=None, labels=None, infer: bool = False, use_cache: bool = False, to_compute_mask=None,
                cat: str = "", **_) -> ModelOutput:
        """`model(input_ids, infer=True, use_cache=False).logits` of the reference wrapper (modeling_xllmx_dimoo.py:41-72). The two
        extra keywords are those of the class underneath it, LLaDAModelLM.forward (modeling_llada.py:1475-1477): with the token
        cache switched on (`caching(True)`) and `use_cache=True` they select the partial-recompute forward."""
        if labels is not None or not infer:
            raise NotImplementedError("only the inference branch (infer=True) is on the H100 hot path")
        if to_compute_mask is not None and not (use_cache and getattr(self, "_caching", False)):
            raise ValueError("to_compute_mask needs the token cache: model.caching(True) and use_cache=True")
        # use_cache=True with the cache switched on and no mask: a full forward that fills the caches (same logits);
        # with the cache off the flag is output-invariant (the reference's stores are then never read).
        ids = self._ids_device(input_ids)
        B, L = ids.shape
        if use_cache and getattr(self, "_caching", False):
            return ModelOutput(logits=self._forward_cached(ids, to_compute_mask, cat), attn_key_values=None, hidden_states=None)
        logits = torch.empty((B, L, self.vocab_rows), dtype=torch.bfloat16, device=self.device)
        check(lib.mmdp_model_forward(self._h, ptr(ids), B, L, ptr(logits), None, 0, None, None, 0, 0, 0, None, stream_ptr()))
        return ModelOutput(logits=logits, attn_key_values=None, hidden_states=None)

    __call__ = forward

    def forward_rows(self, ids: torch.Tensor, rows_a: Optional[torch.Tensor] = None, rows_b: Optional[torch.Tensor] = None,
                     col0_b: int = 0, ncols_b: int = 0, out_a: Optional[torch.Tensor] = None,
                     out_b: Optional[torch.Tensor] = None, row_window: Optional[tuple] = None):
        """One forward over ids [B, L] (cuda int64). rows_* are int32 flattened row indices b*L + pos.
        Returns (logits_a [n_a, V] or None, logits_b [n_b, ncols_b] or None).
        row_window = (lo, hi): every requested row is a position in [lo, hi) of its batch row - the last block then computes its
        attention output and MLP for those positions only (keys / values for all rows): nothing after it mixes rows, the skipped
        rows are never read. A row outside the window raises IndexError at the next raise_device_errors()."""
        B, L = ids.shape
        n_a = 0 if rows_a is None else rows_a.numel()
        n_b = 0 if rows_b is None else rows_b.numel()
        if n_a and out_a is None:
            out_a = torch.empty((n_a, self.vocab_rows), dtype=torch.bfloat16, device=self.device)
        if n_b and out_b is None:
            out_b = torch.empty((n_b, ncols_b), dtype=torch.bfloat16, device=self.device)
        lo, hi = (int(row_window[0]), int(row_window[1])) if row_window is not None else (0, 0)
        check(lib.mmdp_model_forward_window(self._h, ptr(ids), B, L, ptr(rows_a), n_a, ptr(out_a) if n_a else None,
                                            ptr(rows_b), n_b, col0_b, ncols_b, ptr(out_b) if n_b else None, lo, hi, stream_ptr()))
        return (out_a if n_a else None), (out_b if n_b else None)
