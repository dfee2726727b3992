"""Shared helpers for the test-suite (tests may import oracle/; product code may not)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def tiny_cfg_and_weights(meta):
    from oracle import llada
    cfg = llada.make_config(**meta["tiny"])
    sd = llada.make_weights(cfg, seed=meta["weight_seed"])
    return cfg, sd


_TINY_CACHE = {}


def tiny_gpu_model(meta, cls=None, max_batch=3):
    """H100-native model with the deterministic tiny weights of the golden fixtures (cached per process)."""
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
    cls = cls or LLaDAForMultiModalGeneration
    key = (cls.__name__, meta["weight_seed"], tuple(sorted(meta["tiny"].items())), max_batch)
    if key not in _TINY_CACHE:
        cfg, sd = tiny_cfg_and_weights(meta)
        if cls.__name__ == "MMadaModelLM":
            cfg.mask_token_id = 126336
        m = cls(cfg, max_seq_len=cfg.max_sequence_length, max_batch=max_batch)
        m.load_state_dict(sd)
        _TINY_CACHE[key] = (m, cfg, sd)
    return _TINY_CACHE[key]


class GpuBackedOracleModel:
    """Oracle-side model whose logits come from the H100 forward (full LM head), moved to the CPU. Lets the CPU oracle
    loop run on exactly the logits the CUDA sampling kernels see, so integer decisions must agree bit-for-bit."""

    def __init__(self, gpu_model):
        self.m = gpu_model
        self.device = torch.device("cpu")

    def __call__(self, input_ids, infer=True, use_cache=False, **_):
        from types import SimpleNamespace
        out = self.m(input_ids, infer=True, use_cache=False).logits
        return SimpleNamespace(logits=out.cpu())


def bf16_ulp_err(got, want):
    """Max error in units of the bf16 spacing at the magnitude of `want` (floor 2^-126)."""
    g, w = got.float(), want.float()
    ulp = torch.maximum(w.abs(), torch.tensor(1e-30)).log2().floor().exp2() * 2.0 ** -7
    return ((g - w).abs() / ulp).max().item()
