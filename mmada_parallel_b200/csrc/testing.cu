// Test hooks (include/mmdp_testing.h: the VQ kernels; include/mmdp_testing_cache.h: the token-cache launches): internal kernels
// behind thin C wrappers, so that tests can check each operation against a high-precision restatement of it. Each hook forwards
// its arguments unchanged.
#include "../../include/mmdp_testing.h"
#include "../../include/mmdp_testing_cache.h"
#include "mmdp_internal.h"

using namespace mmdp;

namespace {
int need_device(const char* fn) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return set_error("%s: no CUDA device (this library has no CPU fallback)", fn);
    return 0;
}
}  // namespace

extern "C" {

MMDP_API int mmdp_testing_conv_tf32(const float* A, int lda, long long a_rows, const float* W, int M, int N, int K, int T,
                                    const int* shifts_host, float* C, int ldc, const float* R, int ldr, const float* bias,
                                    int bias_along_m, float alpha, int pad_w, int pad_h, int scatter_w, int scatter_h,
                                    void* stream) {
    if (need_device(__func__)) return -1;
    return conv_tf32(A, lda, a_rows, W, M, N, K, T, shifts_host, C, ldc, R, ldr, bias, bias_along_m, alpha, pad_w, pad_h,
                     scatter_w, scatter_h, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_gn_swish(const float* x, float* y, int B, int C, int H, int W, double* stats_ws, const float* gamma,
                                   const float* beta, float eps, int swish, int compact, void* stream) {
    if (need_device(__func__)) return -1;
    return gn_swish(x, y, B, C, H, W, stats_ws, gamma, beta, eps, swish, compact, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_upsample2x(const float* x, float* y, int B, int C, int H, int W, void* stream) {
    if (need_device(__func__)) return -1;
    return upsample2x(x, y, B, C, H, W, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_downsample_pick(const float* src, float* dst, int B, int C, int H, int W, void* stream) {
    if (need_device(__func__)) return -1;
    return downsample_pick(src, dst, B, C, H, W, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_softmax_rows_ld(float* s, int rows, int n, int ld, void* stream) {
    if (need_device(__func__)) return -1;
    return softmax_rows_ld(s, rows, n, ld, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_zero_border(float* y, int B, int C, int H, int W, void* stream) {
    if (need_device(__func__)) return -1;
    return zero_border(y, B, C, H, W, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_nchw_to_padded(const float* x, float* y, int B, int C, int Cpad, int H, int W, void* stream) {
    if (need_device(__func__)) return -1;
    return nchw_to_padded(x, y, B, C, Cpad, H, W, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_padded_to_nchw(const float* x, float* y, int B, int C, int ld, int H, int W, void* stream) {
    if (need_device(__func__)) return -1;
    return padded_to_nchw(x, y, B, C, ld, H, W, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_lfq_to_padded(const int64_t* ids, float* z, int B, int H, int W, int bits, int Cpad, void* stream) {
    if (need_device(__func__)) return -1;
    return lfq_to_padded(ids, z, B, H, W, bits, Cpad, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_lfq_indices(const float* z, int64_t* ids, int B, int h, int w, int bits, int ld, void* stream) {
    if (need_device(__func__)) return -1;
    return lfq_indices(z, ids, B, h, w, bits, ld, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_codebook_to_padded(const int64_t* ids, const float* cb, float* z, int B, int h, int w, int C, int Cpad,
                                             int64_t n_codes, int* err, void* stream) {
    if (need_device(__func__)) return -1;
    return codebook_to_padded(ids, cb, z, B, h, w, C, Cpad, n_codes, err, (cudaStream_t)stream);
}

MMDP_API int mmdp_testing_qkv_rope_cached(int precision, const void* A, int lda, const float* sa, const void* Wqkv, const float* sw,
                                          int B, int Tq, const int32_t* pos_map, int d_model, int n_heads, int L, int Lpad,
                                          const float* cos, const float* sin, uint16_t* q, uint16_t* kcache, uint16_t* vtcache,
                                          void* stream) {
    if (need_device(__func__)) return -1;
    QkvRopeArgs qa{(__nv_bfloat16*)q, (__nv_bfloat16*)kcache, (__nv_bfloat16*)vtcache, cos, sin, L, Lpad, d_model, n_heads,
                   pos_map, pos_map ? Tq : 0};
    const int M = B * Tq, N = 3 * d_model;
    if (precision == 0)
        return gemm_bf16(EPI_QKVROPE, (const __nv_bfloat16*)A, lda, (const __nv_bfloat16*)Wqkv, d_model, M, N, d_model, nullptr, 0,
                         nullptr, 0, &qa, (cudaStream_t)stream);
    if (precision == 1)
        return gemm_fp8(EPI_QKVROPE, (const uint8_t*)A, lda, sa, (const uint8_t*)Wqkv, d_model, sw, M, N, d_model, nullptr, 0, nullptr,
                        0, &qa, (cudaStream_t)stream);
    return set_error("%s: precision %d is neither 0 (bf16) nor 1 (e4m3)", __func__, precision);
}

MMDP_API int mmdp_testing_attention_cached(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, int H,
                                           int L, int Lpad, int Tq, float scale, void* stream) {
    if (need_device(__func__)) return -1;
    return attention_fwd((const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)vt, (__nv_bfloat16*)out, B, H, L, Lpad,
                         scale, (cudaStream_t)stream, Tq);
}

}  // extern "C"
