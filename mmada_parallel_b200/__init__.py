"""mmada_parallel_b200 - H100-native (sm_90a) implementation of the MMaDA-Parallel parallel-denoising hot path.

Public surface mirrors the reference's inference API for that path only:
  mmada_parallel_b200.model.LLaDAForMultiModalGeneration        (A/model/modeling_xllmx_dimoo.py)
  mmada_parallel_b200.generators.parallel_generator.generate_ti2ti   (A/generators/parallel_generator.py)
  mmada_parallel_b200.mmada.MMadaModelLM.interleave_generate    (M/models/modeling_mmada.py)
  mmada_parallel_b200.magvit.MAGVITv2.decode_code               (M/models/modeling_magvitv2.py)
All compute goes through libmmdp.so (C ABI in include/mmdp.h); importing this package without the built library
raises ImportError - there is no CPU fallback.
"""
from . import _lib  # noqa: F401  (fails loudly if libmmdp.so is missing)

__version__ = "0.1.0"
