"""Loader for the REAL reference (read-only import from the checkout named by MMDP_REFERENCE_ROOT). Used ONLY by
oracle/make_golden*.py to pin the oracle and write the golden fixtures; nothing under tests, smoke() or bench.py may import
this module, so the suite runs without the reference.

Recipes follow SURVEY.md §8c. No reference source is copied; modules are imported where they lie, with
PYTHONDONTWRITEBYTECODE so nothing is written into the read-only tree.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REF_ROOT = os.environ.get("MMDP_REFERENCE_ROOT", "")  # a checkout of tyfeld/MMaDA-Parallel
REF_A = os.path.join(REF_ROOT, "MMaDA-Parallel-A")
REF_M = os.path.join(REF_ROOT, "MMaDA-Parallel-M")

sys.dont_write_bytecode = True


def available() -> bool:
    return bool(REF_ROOT) and os.path.isdir(REF_A) and os.path.isdir(REF_M)


def load_a():
    """Returns (LLaDAForMultiModalGeneration, LLaDAConfig, parallel_generator module, modeling_llada module)."""
    if REF_A not in sys.path:
        sys.path.insert(0, REF_A)
    from model import LLaDAForMultiModalGeneration  # noqa
    from model.configuration_llada import LLaDAConfig  # noqa
    import model.modeling_llada as modeling_llada  # noqa
    pg = importlib.import_module("generators.parallel_generator")
    return LLaDAForMultiModalGeneration, LLaDAConfig, pg, modeling_llada


def ref_config_a(cfg):
    """LLaDAConfig carrying the fields of oracle.llada.make_config(...)."""
    _, LLaDAConfig, _, _ = load_a()
    return LLaDAConfig(
        d_model=cfg.d_model, n_heads=cfg.n_heads, n_layers=cfg.n_layers, mlp_hidden_size=cfg.mlp_hidden_size,
        vocab_size=cfg.vocab_size, embedding_size=cfg.embedding_size, rope_theta=cfg.rope_theta,
        rms_norm_eps=cfg.rms_norm_eps, max_sequence_length=cfg.max_sequence_length, block_type="llama",
        activation_type="silu", layer_norm_type="rms", rope=True, rope_full_precision=True, weight_tying=False,
        include_bias=False, attention_dropout=0.0, residual_dropout=0.0, embedding_dropout=0.0, alibi=False,
        layer_norm_with_affine=True, attention_layer_norm=False, init_device="cpu", flash_attention=False,
        scale_logits=False, input_emb_norm=False, block_group_size=1, n_kv_heads=None, multi_query_attention=None,
    )


def build_ref_model_a(cfg, state_dict):
    import torch
    Model, _, _, _ = load_a()
    m = Model(ref_config_a(cfg), init_params=False).eval()
    m = m.to(torch.bfloat16)
    missing, unexpected = m.load_state_dict(state_dict, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in k or "inv_freq" in k for k in missing), missing
    return m


def load_m():
    """Returns the modules (modeling_mmada, sampling, modeling_magvitv2) of variant M, bypassing the package __init__
    that imports a file missing from the reference (models/__init__.py:1)."""
    if "models" not in sys.modules or getattr(sys.modules["models"], "__path__", None) != [os.path.join(REF_M, "models")]:
        pkg = types.ModuleType("models")
        pkg.__path__ = [os.path.join(REF_M, "models")]
        sys.modules["models"] = pkg
    # stubs for packages that are absent in this image and unused on the path
    if "omegaconf" not in sys.modules:
        oc = types.ModuleType("omegaconf")
        oc.OmegaConf = type("OmegaConf", (), {})
        oc.DictConfig = dict
        oc.ListConfig = list
        sys.modules["omegaconf"] = oc
    if "models.modeling_utils" not in sys.modules:
        import torch.nn as nn
        mu = types.ModuleType("models.modeling_utils")
        mu.ModelMixin = nn.Module
        mu.ConfigMixin = object
        mu.register_to_config = lambda f: f
        sys.modules["models.modeling_utils"] = mu
    mm = importlib.import_module("models.modeling_mmada")
    sm = importlib.import_module("models.sampling")
    try:
        mv = importlib.import_module("models.modeling_magvitv2")
    except Exception:  # pragma: no cover - magvit import is optional for the sampler fixtures
        mv = None
    return mm, sm, mv


def load_app():
    """MMaDA-Parallel-A/app.py (Gradio demo) with its UI / diffusers imports stubbed: the module builds its Blocks at import
    time, so `gradio` is a MagicMock; `utils.image_utils` imports diffusers at module level."""
    from unittest.mock import MagicMock
    if REF_A not in sys.path:
        sys.path.insert(0, REF_A)
    sys.modules.setdefault("gradio", MagicMock())
    if "diffusers" not in sys.modules:
        d = types.ModuleType("diffusers")
        d.VQModel = object
        dp = types.ModuleType("diffusers.image_processor")
        dp.VaeImageProcessor = object
        sys.modules["diffusers"] = d
        sys.modules["diffusers.image_processor"] = dp
    return importlib.import_module("app")
