/*
 * mmdp_testing.h - test hooks of libmmdp.so: the internal kernels of the VQ tokenizers (csrc/conv_tf32.cu,
 * csrc/vq_codebook.cu), exported one by one so that a test can compare each operation with a high-precision
 * restatement of it. Not part of the product ABI in mmdp.h: no product code calls these, and their signatures follow
 * the internal functions in csrc/mmdp_internal.h rather than a stability promise.
 *
 * Every hook only forwards its arguments to the internal function of the same name (conventions as in mmdp.h: device
 * pointers, 0 / -1 return with mmdp_last_error(), `stream` a cudaStream_t as void*). Without a CUDA device every hook
 * returns -1 before it touches a pointer.
 */
#ifndef MMDP_TESTING_H_
#define MMDP_TESTING_H_

#include "mmdp.h"

#ifdef __cplusplus
extern "C" {
#endif

/* TF32 shifted-tap GEMM: C[m, n] = alpha * sum_{t < T} sum_k A[m + shifts_host[t], k] * W[t*N + n, k] + bias (+ R[m, n]).
 * A [a_rows, lda] fp32 (rows outside [0, a_rows) read as zero), W [T*N, K] fp32, K a multiple of 32. pad_w > 0: rows index
 * padded images of pad_h x pad_w pixels and border rows are written as zero; scatter_w > 0: rows index compact
 * scatter_h x scatter_w images and C / R rows live in the padded layout of those images. bias_along_m: bias[m]. */
MMDP_API int mmdp_testing_conv_tf32(const float* A, int lda, long long a_rows, const float* W, int M, int N, int K, int T,
                                    const int* shifts_host, float* C, int ldc, const float* R, int ldr, const float* bias,
                                    int bias_along_m, float alpha, int pad_w, int pad_h, int scatter_w, int scatter_h,
                                    void* stream);
/* GroupNorm(32 groups) (+ SiLU) of padded NHWC x [B, (H+2)(W+2), C]; stats_ws: B * 64 doubles of workspace.
 * compact == 0: padded y with a zero border; compact == 1: y [B, H*W, C]. */
MMDP_API int mmdp_testing_gn_swish(const float* x, float* y, int B, int C, int H, int W, double* stats_ws, const float* gamma,
                                   const float* beta, float eps, int swish, int compact, void* stream);
MMDP_API int mmdp_testing_upsample2x(const float* x, float* y, int B, int C, int H, int W, void* stream);
MMDP_API int mmdp_testing_downsample_pick(const float* src, float* dst, int B, int C, int H, int W, void* stream);
MMDP_API int mmdp_testing_softmax_rows_ld(float* s, int rows, int n, int ld, void* stream);
MMDP_API int mmdp_testing_zero_border(float* y, int B, int C, int H, int W, void* stream);
MMDP_API int mmdp_testing_nchw_to_padded(const float* x, float* y, int B, int C, int Cpad, int H, int W, void* stream);
MMDP_API int mmdp_testing_padded_to_nchw(const float* x, float* y, int B, int C, int ld, int H, int W, void* stream);
MMDP_API int mmdp_testing_lfq_to_padded(const int64_t* ids, float* z, int B, int H, int W, int bits, int Cpad, void* stream);
MMDP_API int mmdp_testing_lfq_indices(const float* z, int64_t* ids, int B, int h, int w, int bits, int ld, void* stream);
/* err: device int, bit 0 raised by an id outside [0, n_codes) */
MMDP_API int mmdp_testing_codebook_to_padded(const int64_t* ids, const float* cb, float* z, int B, int h, int w, int C, int Cpad,
                                             int64_t n_codes, int* err, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* MMDP_TESTING_H_ */
