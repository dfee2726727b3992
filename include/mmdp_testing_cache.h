/*
 * mmdp_testing_cache.h - test hooks of libmmdp.so for the two launch forms of the token-cache forward
 * (mmdp_model_forward_cached): the QKV + RoPE GEMM with a position map and attention of Tq query rows against L cached keys,
 * exported so that a test can compare each with a high-precision restatement of it. Same status and conventions as the VQ
 * hooks of mmdp_testing.h: not part of the product ABI in mmdp.h, signatures follow the internal functions in
 * csrc/mmdp_internal.h, every hook only forwards its arguments and returns -1 without a CUDA device.
 */
#ifndef MMDP_TESTING_CACHE_H_
#define MMDP_TESTING_CACHE_H_

#include "mmdp.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Token-cache QKV + RoPE (gemm_bf16 / gemm_fp8 with EPI_QKVROPE): A [B*Tq, d_model] (lda), Wqkv [3 d_model, d_model]; compact
 * row r is token pos_map[r] of batch row r / Tq. q [B*Tq, d_model] stays compact; k rows go to kcache [B*L, d_model] at
 * b*L + pos and V^T columns to vtcache [B, n_heads, 128, Lpad] at pos. pos_map == NULL with Tq == L is the full forward.
 * precision 0: bf16 operands (sa, sw ignored); 1: e4m3 operands, sa [d_model / 128][B*Tq] and sw [3 d_model] fp32 scales. */
MMDP_API int mmdp_testing_qkv_rope_cached(int precision, const void* A, int lda, const float* sa, const void* Wqkv, const float* sw,
                                          int B, int Tq, const int32_t* pos_map, int d_model, int n_heads, int L, int Lpad,
                                          const float* cos, const float* sin, uint16_t* q, uint16_t* kcache, uint16_t* vtcache,
                                          void* stream);
/* attention_fwd with Lq = Tq: q / out [B*Tq, 128 H], k [B*L, 128 H], vt [B, H, 128, Lpad] (columns [L, Lpad) zero) */
MMDP_API int mmdp_testing_attention_cached(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, int H,
                                           int L, int Lpad, int Tq, float scale, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* MMDP_TESTING_CACHE_H_ */
