"""ctypes binding of libmmdp.so (the C ABI declared in include/mmdp.h).

The library is the product path: there is no Python/torch fallback for any op. If the shared object is
missing the import raises; if a call is made without a CUDA device the C side returns an error that is
re-raised here as RuntimeError.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmmdp.so")

EPI_PLAIN, EPI_RESID, EPI_SWIGLU, EPI_F32 = 0, 1, 3, 4
PRECISION_BF16, PRECISION_FP8 = 0, 1
ARCH_QKV_BIAS = 1  # mmdp_model_create_arch flags


class MmdpError(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C mmada_parallel_b200/csrc`). This package has no CPU fallback."
        )
    return C.CDLL(LIB_PATH)


lib = _load()

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float


class VqDecConfig(C.Structure):
    _fields_ = [("ch", C.c_int32), ("n_levels", C.c_int32), ("ch_mult", C.c_int32 * 8), ("num_res_blocks", C.c_int32 * 8),
                ("z_channels", C.c_int32), ("out_ch", C.c_int32), ("max_batch", C.c_int32), ("latent_h", C.c_int32),
                ("latent_w", C.c_int32)]


class VqModelConfig(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("out_channels", C.c_int32), ("n_levels", C.c_int32),
                ("block_out_channels", C.c_int32 * 8), ("layers_per_block", C.c_int32), ("latent_channels", C.c_int32),
                ("num_vq_embeddings", C.c_int32), ("mid_block_add_attention", C.c_int32), ("max_batch", C.c_int32),
                ("max_latent_cells", C.c_int32)]


class TpLayer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("wqkv", "wo", "w13", "w2", "attn_norm", "ff_norm", "bqkv")]


class TpLayerFp8(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("wqkv", "wo", "w13", "w2", "sqkv", "so", "s13", "s2")]


class TpChunk(C.Structure):
    _fields_ = [("x_shard", C.c_void_p), ("recv", C.POINTER(C.c_void_p) * 2), ("flags", C.POINTER(C.c_void_p)), ("done_counter", C.c_void_p)]


class TpPacked(C.Structure):
    """mmdp_tp_ctx.packed: the device row map int2 [max_rows] of packed forwards and the capacities it is checked against."""
    _fields_ = [("seg_pos", C.c_void_p), ("max_rows", C.c_int32), ("rope_len", C.c_int32)]


class TpCtx(C.Structure):
    _fields_ = [("d_model", C.c_int32), ("n_heads_local", C.c_int32), ("ff_local", C.c_int32), ("n_layers", C.c_int32),
                ("n_ranks", C.c_int32), ("rank", C.c_int32), ("rms_eps", C.c_float), ("layers", C.POINTER(TpLayer)),
                ("wte", C.c_void_p), ("ln_f", C.c_void_p), ("vocab", C.c_int64), ("cos_tab", C.c_void_p), ("sin_tab", C.c_void_p),
                ("q", C.c_void_p), ("k", C.c_void_p), ("att", C.c_void_p), ("h", C.c_void_p), ("vt", C.c_void_p),
                ("xn", C.POINTER(C.c_void_p)), ("n_chunks", C.c_int32), ("chunk_rows0", C.c_int32), ("chunk", TpChunk * 2),
                ("n_kv_heads_local", C.c_int32), ("precision", C.c_int32), ("layers_fp8", C.POINTER(TpLayerFp8)),
                ("xq", C.POINTER(C.c_void_p)), ("xq_scales", C.POINTER(C.c_void_p)), ("a8", C.c_void_p), ("a8_scales", C.c_void_p),
                ("packed", TpPacked)]


class ModelConfig(C.Structure):
    _fields_ = [
        ("d_model", C.c_int32),
        ("n_heads", C.c_int32),
        ("n_layers", C.c_int32),
        ("mlp_hidden", C.c_int32),
        ("vocab_size", C.c_int32),
        ("max_seq_len", C.c_int32),
        ("max_batch", C.c_int32),
        ("rms_eps", C.c_float),
    ]


# name -> (restype, argtypes); must list every symbol declared in include/mmdp.h (checked by tests/test_abi.py)
SIGNATURES = {
    "mmdp_version": (_i, []),
    "mmdp_last_error": (C.c_char_p, []),
    "mmdp_prof_enable": (None, [_i]),
    "mmdp_prof_summary": (_i, [_vp, _vp, _vp]),
    "mmdp_launch_count": (C.c_longlong, [_i]),
    "mmdp_set_gemm_pair": (None, [_i]),
    "mmdp_set_gemm_splitk": (None, [_i]),
    "mmdp_set_pdl": (None, [_i]),
    "mmdp_set_option": (_i, [C.c_char_p, _i]),
    "mmdp_tp_alloc": (_i, [C.c_uint64, C.POINTER(_vp)]),
    "mmdp_tp_free": (_i, [_vp]),
    "mmdp_ipc_export": (_i, [_vp, _vp]),
    "mmdp_ipc_import": (_i, [_vp, C.POINTER(_vp)]),
    "mmdp_ipc_close": (_i, [_vp]),
    "mmdp_tp_forward": (_i, [C.POINTER(TpCtx), _vp, _i, _i, C.c_uint32, C.POINTER(C.c_uint32), _vp]),
    "mmdp_tp_forward_packed": (_i, [C.POINTER(TpCtx), _vp, _i, _vp, C.c_uint32, C.POINTER(C.c_uint32), _vp]),
    "mmdp_gemm_f32_scatter": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "mmdp_tp_reduce_norm": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _f, C.c_uint32, _vp, _vp]),
    "mmdp_gemm_fp8_f32": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _i, _i, _vp, _i, _vp]),
    "mmdp_gemm_fp8_f32_scatter": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "mmdp_tp_reduce_norm_fp8": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp, _i, _i, _vp, _vp, _i, _i, _i, _f, C.c_uint32, _vp, _vp]),
    "mmdp_gemm_bf16": (_i, [_i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp]),
    "mmdp_quantize_fp8": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp]),
    "mmdp_gemm_fp8": (_i, [_i, _vp, _i, _vp, _vp, _i, _vp, _i, _i, _i, _vp, _i, _vp, _i, _vp]),
    "mmdp_qkv_rope": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_qkv_rope_tp": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_qkv_rope_gqa": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_qkv_rope_tp_gqa": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_qkv_rope_tp_fp8": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_qkv_rope_tp_packed": (_i, [_i, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_resid_add_f32": (_i, [_vp, _i, _vp, _i, _i, _i, _vp]),
    "mmdp_attention": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    "mmdp_attention_packed": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _f, _vp]),
    "mmdp_attention_packed_window": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _f, _vp]),
    "mmdp_attention_gqa": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _f, _vp]),
    "mmdp_rmsnorm": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _f, _vp]),
    "mmdp_embed": (_i, [_vp, _vp, _vp, _i, _i, _i64, _vp]),
    "mmdp_text_step": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _i64, _f, _vp, _i64, _i, _vp, _vp, _vp]),
    "mmdp_text_step_gumbel64": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _i64, _f, _vp, _i64, _i, _vp, _vp, _vp]),
    "mmdp_image_step_t2i": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _f, _vp, _f, _i, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_image_step": (
        _i,
        [_i, _vp, _vp, _vp, _i64, _i, _i, _f, _f, _vp, _vp, _f, _i, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    ),
    "mmdp_image_remask": (_i, [_i, _i, _vp, _vp, _vp, _vp, _f, _i, _vp, _vp, _i64, _i64, _vp, _vp, _vp]),
    "mmdp_lfq_decode": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "mmdp_vqdec_create": (_i, [C.POINTER(VqDecConfig), C.POINTER(_vp)]),
    "mmdp_vqdec_destroy": (None, [_vp]),
    "mmdp_vqdec_set_weight": (_i, [_vp, C.c_char_p, _vp, _i64, _vp]),
    "mmdp_vqdec_missing": (_i, [_vp, C.c_char_p, _i]),
    "mmdp_vqdec_decode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_vqenc_create": (_i, [C.POINTER(VqDecConfig), C.POINTER(_vp)]),
    "mmdp_vqenc_encode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_vqmodel_create": (_i, [C.POINTER(VqModelConfig), C.POINTER(_vp)]),
    "mmdp_vqmodel_decode": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_vqmodel_encode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_vqmodel_error_flags": (_i, [_vp, C.POINTER(C.c_int32), _vp]),
    "mmdp_vq_nearest": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "mmdp_model_create": (_i, [C.POINTER(ModelConfig), C.POINTER(_vp)]),
    "mmdp_model_create_ex": (_i, [C.POINTER(ModelConfig), _i, C.POINTER(_vp)]),
    "mmdp_model_create_arch": (_i, [C.POINTER(ModelConfig), _i, _i, _i, C.POINTER(_vp)]),
    "mmdp_model_destroy": (None, [_vp]),
    "mmdp_model_set_weight": (_i, [_vp, C.c_char_p, _vp, _i64, _i64, _vp]),
    "mmdp_model_set_rope": (_i, [_vp, _vp, _vp, _i, _vp]),
    "mmdp_model_forward": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_model_forward_window": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _vp]),
    "mmdp_model_forward_packed": (_i, [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_model_forward_packed_window": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "mmdp_model_forward_cached": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "mmdp_model_hidden": (_vp, [_vp]),
    "mmdp_model_error_flags": (_i, [_vp, C.POINTER(C.c_int32), _vp]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)
    _fn.restype = _res
    _fn.argtypes = _args


def check(rc: int) -> None:
    if rc != 0:
        raise MmdpError(lib.mmdp_last_error().decode("utf-8", "replace"))


def prof_summary():
    """{kind: (ms, work, launches)} accumulated since mmdp_prof_enable(1); synchronises the device."""
    ms, work, n = (C.c_double * 4)(), (C.c_double * 4)(), (C.c_longlong * 4)()
    check(lib.mmdp_prof_summary(ms, work, n))
    return {k: (ms[i], work[i], n[i]) for i, k in enumerate(("gemm", "attention", "row", "sampling"))}


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Raw device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream_ptr() -> Optional[int]:
    """The current torch CUDA stream as a cudaStream_t."""
    if not torch.cuda.is_available():
        return None
    return torch.cuda.current_stream().cuda_stream or None


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise MmdpError("mmada_parallel_b200: tensors must live on a CUDA device (no CPU fallback)")


# ---------------------------------------------------------------------------------------------------------------
# thin op wrappers (used by the tests and by the host-side generators)
# ---------------------------------------------------------------------------------------------------------------
def gemm_bf16(a: torch.Tensor, w: torch.Tensor, epilogue: int = EPI_PLAIN, resid: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C = A @ W^T with a fused epilogue. a [M,K], w [N,K] (nn.Linear layout), both bf16 contiguous rows."""
    require_cuda(a, w, resid, out)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=a.device)
    check(lib.mmdp_gemm_bf16(epilogue, ptr(a), a.stride(0), ptr(w), w.stride(0), M, N, K, ptr(out), out.stride(0),
                             ptr(resid), resid.stride(0) if resid is not None else 0, stream_ptr()))
    return out


def quantize_fp8(x: torch.Tensor, group: int = 128):
    """e4m3 quantisation of a bf16 [rows, K] tensor (row stride may exceed K) in row groups of `group` elements.
    Returns (q float8_e4m3fn [rows, K], scales fp32 [K // group, rows])."""
    require_cuda(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    rows, K = x.shape
    q = torch.empty((rows, K), dtype=torch.float8_e4m3fn, device=x.device)
    s = torch.empty((K // group, rows), dtype=torch.float32, device=x.device)
    check(lib.mmdp_quantize_fp8(ptr(x), x.stride(0), rows, K, group, ptr(q), K, ptr(s), stream_ptr()))
    return q, s


def gemm_fp8(qa: torch.Tensor, sa: torch.Tensor, qw: torch.Tensor, sw: torch.Tensor, epilogue: int = EPI_PLAIN,
             resid: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C = epilogue(sw[n] * sum_g sa[g, m] * (qa[m, g] . qw[n, g])): qa [M, K] e4m3 with scales sa [K/128, M], qw [N, K] e4m3
    with row scales sw [N]. For EPI_SWIGLU the gate / up rows of qw (and sw) are interleaved in 64-row blocks."""
    require_cuda(qa, sa, qw, sw, resid, out)
    assert qa.dtype == torch.float8_e4m3fn and qw.dtype == torch.float8_e4m3fn
    assert sa.dtype == torch.float32 and sw.dtype == torch.float32 and sa.is_contiguous() and sw.is_contiguous()
    M, K = qa.shape
    N = qw.shape[0]
    assert tuple(sa.shape) == (K // 128, M) and tuple(sw.shape) == (N,)
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=qa.device)
    check(lib.mmdp_gemm_fp8(epilogue, ptr(qa), qa.stride(0), ptr(sa), ptr(qw), qw.stride(0), ptr(sw), M, N, K, ptr(out),
                            out.stride(0), ptr(resid), resid.stride(0) if resid is not None else 0, stream_ptr()))
    return out


def qkv_rope(a: torch.Tensor, wqkv: torch.Tensor, n_heads: int, L: int, cos: torch.Tensor, sin: torch.Tensor):
    require_cuda(a, wqkv, cos, sin)
    M, d = a.shape
    B = M // L
    Lpad = (L + 7) // 8 * 8
    q = torch.empty((M, d), dtype=torch.bfloat16, device=a.device)
    k = torch.empty((M, d), dtype=torch.bfloat16, device=a.device)
    vt = torch.zeros((B, n_heads, 128, Lpad), dtype=torch.bfloat16, device=a.device)
    check(lib.mmdp_qkv_rope(ptr(a), a.stride(0), ptr(wqkv), M, d, n_heads, L, Lpad, ptr(cos), ptr(sin), ptr(q), ptr(k),
                            ptr(vt), stream_ptr()))
    return q, k, vt


def attention(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, B: int, n_heads: int, L: int, scale: float) -> torch.Tensor:
    require_cuda(q, k, vt)
    out = torch.empty_like(q)
    check(lib.mmdp_attention(ptr(q), ptr(k), ptr(vt), ptr(out), B, n_heads, L, vt.shape[-1], scale, stream_ptr()))
    return out


def attention_packed(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, seq_lens, n_heads: int, scale: float) -> torch.Tensor:
    """Attention over a packed batch: q, k [sum(seq_lens), n_heads * 128]; vt [len(seq_lens), n_heads, 128, Lpad] with zero
    (or finite) pad columns. Each sequence attends to its own keys only."""
    require_cuda(q, k, vt)
    lens = (C.c_int32 * len(seq_lens))(*[int(x) for x in seq_lens])
    out = torch.empty_like(q)
    check(lib.mmdp_attention_packed(ptr(q), ptr(k), ptr(vt), ptr(out), len(seq_lens), lens, n_heads, vt.shape[-1], scale,
                                    stream_ptr()))
    return out


def attention_packed_window(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, seq_lens, windows, n_heads: int, scale: float,
                            n_kv_heads: int = 0) -> torch.Tensor:
    """Packed attention for the query rows [lo, hi) of every sequence only: windows = [(lo, hi)] per sequence. q [sum(seq_lens),
    n_heads * 128], k [sum(seq_lens), n_kv_heads * 128] and vt [len(seq_lens), n_kv_heads, 128, Lpad] as in attention_packed
    (n_kv_heads 0: n_heads). Returns the windows' rows end to end, [sum(hi - lo), n_heads * 128]."""
    require_cuda(q, k, vt)
    n = len(seq_lens)
    lens = (C.c_int32 * n)(*[int(x) for x in seq_lens])
    lo = (C.c_int32 * n)(*[int(w[0]) for w in windows])
    hi = (C.c_int32 * n)(*[int(w[1]) for w in windows])
    out = torch.empty((sum(int(w[1]) - int(w[0]) for w in windows), q.shape[1]), dtype=q.dtype, device=q.device)
    check(lib.mmdp_attention_packed_window(ptr(q), ptr(k), ptr(vt), ptr(out), n, lens, lo, hi, n_heads, n_kv_heads or n_heads,
                                           vt.shape[-1], scale, stream_ptr()))
    return out


def qkv_rope_gqa(a: torch.Tensor, wqkv: torch.Tensor, bias: Optional[torch.Tensor], n_heads: int, n_kv_heads: int, L: int,
                 cos: torch.Tensor, sin: torch.Tensor):
    """Grouped-query q/k/v projection + RoPE: wqkv [d + 2 d_kv, d], bias (optional) [d + 2 d_kv] -> q [M, d], k [M, d_kv],
    vt [B, n_kv_heads, 128, Lpad] (pad columns zero)."""
    require_cuda(a, wqkv, bias, cos, sin)
    M, d = a.shape
    B = M // L
    Lpad = (L + 7) // 8 * 8
    q = torch.empty((M, d), dtype=torch.bfloat16, device=a.device)
    k = torch.empty((M, 128 * n_kv_heads), dtype=torch.bfloat16, device=a.device)
    vt = torch.zeros((B, n_kv_heads, 128, Lpad), dtype=torch.bfloat16, device=a.device)
    check(lib.mmdp_qkv_rope_gqa(ptr(a), a.stride(0), ptr(wqkv), ptr(bias), M, d, n_heads, n_kv_heads, L, Lpad, ptr(cos), ptr(sin),
                                ptr(q), ptr(k), ptr(vt), stream_ptr()))
    return q, k, vt


def attention_gqa(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, n_heads: int, n_kv_heads: int, scale: float, B: int = 1,
                  L: int = 0, seq_lens=None) -> torch.Tensor:
    """Grouped-query attention: q [rows, n_heads * 128], k [rows, n_kv_heads * 128], vt [B or len(seq_lens), n_kv_heads, 128, Lpad].
    seq_lens None: B sequences of L rows; otherwise a packed batch."""
    require_cuda(q, k, vt)
    out = torch.empty_like(q)
    lens = None if seq_lens is None else (C.c_int32 * len(seq_lens))(*[int(x) for x in seq_lens])
    nb = B if seq_lens is None else len(seq_lens)
    check(lib.mmdp_attention_gqa(ptr(q), ptr(k), ptr(vt), ptr(out), nb, lens, n_heads, n_kv_heads, L, vt.shape[-1], scale,
                                 stream_ptr()))
    return out


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, rows: Optional[torch.Tensor] = None) -> torch.Tensor:
    require_cuda(x, w, rows)
    M = x.shape[0] if rows is None else rows.numel()
    d = x.shape[1]
    y = torch.empty((M, d), dtype=torch.bfloat16, device=x.device)
    check(lib.mmdp_rmsnorm(ptr(x), x.stride(0), ptr(rows), ptr(w), ptr(y), d, M, d, eps, stream_ptr()))
    return y


def embed(ids: torch.Tensor, wte: torch.Tensor) -> torch.Tensor:
    require_cuda(ids, wte)
    M = ids.numel()
    x = torch.empty((M, wte.shape[1]), dtype=torch.bfloat16, device=wte.device)
    check(lib.mmdp_embed(ptr(ids), ptr(wte), ptr(x), M, wte.shape[1], wte.shape[0], stream_ptr()))
    return x


def lfq_decode(ids: torch.Tensor, bits: int = 13) -> torch.Tensor:
    require_cuda(ids)
    B, N = ids.shape
    zq = torch.empty((B, bits, N), dtype=torch.float32, device=ids.device)
    check(lib.mmdp_lfq_decode(ptr(ids), ptr(zq), B, N, bits, stream_ptr()))
    return zq
