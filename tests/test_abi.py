"""The C-ABI library loads on a CPU-only box, exports every symbol include/mmdp.h declares, and refuses to compute
without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import torch

from helpers import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "mmdp.h")).read()
    return sorted(set(re.findall(r"MMDP_API[^;(]*?\b(mmdp_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from mmada_parallel_b200 import _lib
    names = declared_symbols()
    assert len(names) >= 16
    for n in names:
        assert hasattr(_lib.lib, n), f"{n} declared in mmdp.h but not exported by libmmdp.so"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in _lib.SIGNATURES"
    assert sorted(_lib.SIGNATURES) == names
    assert _lib.lib.mmdp_version() == 100


def test_no_torch_types_in_header():
    src = open(os.path.join(ROOT, "include", "mmdp.h")).read()
    code = re.sub(r"/\*.*?\*/", "", src, flags=re.S)  # declarations only, comments stripped
    assert "at::" not in code and "torch" not in code.lower() and "Tensor" not in code
    assert "#include <stdint.h>" in code and code.count("#include") == 1


def test_compute_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        return
    from mmada_parallel_b200 import _lib
    cfg = _lib.ModelConfig(256, 2, 2, 512, 134656, 512, 2, 1e-5)
    h = C.c_void_p()
    assert _lib.lib.mmdp_model_create(C.byref(cfg), C.byref(h)) == -1
    assert b"no CUDA device" in _lib.lib.mmdp_last_error()
    # argument validation happens before any device work
    bad = _lib.ModelConfig(200, 2, 2, 512, 134656, 512, 2, 1e-5)
    assert _lib.lib.mmdp_model_create(C.byref(bad), C.byref(h)) == -1
    assert b"head_dim" in _lib.lib.mmdp_last_error()
    try:
        from mmada_parallel_b200.model import LLaDAForMultiModalGeneration
        from oracle.llada import make_config
        LLaDAForMultiModalGeneration(make_config())
        raise AssertionError("model construction must fail without a GPU")
    except _lib.MmdpError as e:
        assert "no CPU fallback" in str(e)


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under the product package may import it."""
    pkg = os.path.join(ROOT, "mmada_parallel_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f"{f} imports oracle"
                assert "/root/reference" not in src


def test_testing_hooks_exported_and_fail_without_gpu():
    """Every hook of include/mmdp_testing.h is exported, kept out of the product table, and errors (not crashes) without a
    device."""
    from mmada_parallel_b200 import _lib
    from test_gpu_vq_ops import HOOKS, declared_testing_symbols, hooks
    names = declared_testing_symbols()
    assert len(names) == 11 and sorted(HOOKS) == names
    lib = hooks()
    for n in names:
        assert n not in _lib.SIGNATURES
    if torch.cuda.is_available():
        return
    for n, args in HOOKS.items():
        zeros = [0.0 if a is C.c_float else None if a is C.c_void_p else 1 for a in args]
        assert getattr(lib, n)(*zeros) == -1, n
        assert b"no CUDA device" in _lib.lib.mmdp_last_error(), n


def test_token_cache_hooks_exported_and_fail_without_gpu():
    """Every hook of include/mmdp_testing_cache.h is exported, kept out of the product table and the VQ hook header, and errors
    (not crashes) without a device."""
    from mmada_parallel_b200 import _lib
    from test_gpu_token_cache import HOOKS, declared_cache_symbols, hooks
    from test_gpu_vq_ops import declared_testing_symbols
    names = declared_cache_symbols()
    assert names == sorted(HOOKS) == ["mmdp_testing_attention_cached", "mmdp_testing_qkv_rope_cached"]
    assert not set(names) & set(declared_testing_symbols())
    lib = hooks()
    for n in names:
        assert n not in _lib.SIGNATURES
    if torch.cuda.is_available():
        return
    for n, args in HOOKS.items():
        zeros = [0.0 if a is C.c_float else None if a is C.c_void_p else 1 for a in args]
        assert getattr(lib, n)(*zeros) == -1, n
        assert b"no CUDA device" in _lib.lib.mmdp_last_error(), n
