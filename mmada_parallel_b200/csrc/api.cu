// extern "C" surface (include/mmdp.h) and the native model context: device-resident packed weights, activation
// workspace and the per-layer launch sequence of LLaDAModel.forward (MMaDA-Parallel-A/model/modeling_llada.py:1201-1415,
// block :906-972). No torch types cross this boundary.
#include "../../include/mmdp.h"
#include "mmdp_internal.h"
#include "ptx.cuh"

#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

using namespace mmdp;
typedef __nv_bfloat16 bf16;

namespace mmdp {

__global__ void lfq_kernel(const int64_t* __restrict__ ids, float* __restrict__ zq, int N, int bits) {
    // z_q[b, c, n] = 2*((id >> (bits-1-c)) & 1) - 1     (LFQuantizer.__init__/get_codebook_entry, modeling_magvitv2.py:186-221)
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int64_t id = ids[(size_t)b * N + n];
    for (int c = 0; c < bits; ++c) zq[((size_t)b * bits + c) * N + n] = ((id >> (bits - 1 - c)) & 1) ? 1.0f : -1.0f;
}

__global__ void packed_row_map_kernel(const __grid_constant__ SegTable segs, int2* __restrict__ seg_pos) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= segs.start[segs.n]) return;
    int s = 0;
    for (int i = 1; i < segs.n; ++i)
        if (r >= segs.start[i]) s = i;
    seg_pos[r] = make_int2(s, r - segs.start[s]);
}

int packed_row_map(const SegTable& segs, int2* seg_pos, cudaStream_t stream) {
    const int M = segs.start[segs.n];
    LaunchScope ls(LK_ROW, 8.0 * M, stream);
    packed_row_map_kernel<<<(M + 255) / 256, 256, 0, stream>>>(segs, seg_pos);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// sequence table of a packed call: n_seg in [1, kMaxSegs], every length in [1, max_len]; returns the longest length, or -1
static int seg_table(const char* who, int n_seg, const int32_t* seg_len, int max_len, SegTable* segs) {
    if (!seg_len || n_seg <= 0 || n_seg > kMaxSegs) return set_error("%s: %d sequences (1 to %d)", who, n_seg, kMaxSegs);
    segs->n = n_seg;
    segs->start[0] = 0;
    int Lmax = 0;
    for (int i = 0; i < n_seg; ++i) {
        if (seg_len[i] <= 0 || seg_len[i] > max_len) return set_error("%s: sequence %d has length %d (1 to %d)", who, i, seg_len[i], max_len);
        segs->start[i + 1] = segs->start[i] + seg_len[i];
        Lmax = seg_len[i] > Lmax ? seg_len[i] : Lmax;
    }
    return Lmax;
}

// Last-block row windows of a packed forward: sequence s (packed rows [start[s], start[s + 1])) keeps its positions [lo[s], hi[s]),
// stored as compact rows [out0[s], out0[s + 1]), the windows of all sequences end to end.
struct WinTable {
    int n;
    int start[kMaxSegs + 1];
    int lo[kMaxSegs], hi[kMaxSegs];
    int out0[kMaxSegs + 1];
};

// xc[j] = x[packed row of compact row j], one CTA per compact row, 16-byte moves
__global__ void __launch_bounds__(128) window_gather_kernel(const __grid_constant__ WinTable w, const bf16* __restrict__ x,
                                                            bf16* __restrict__ xc, int d) {
    const int j = blockIdx.x;
    pdl_launch_dependents();
    pdl_wait();
    int s = 0;
    for (int i = 1; i < w.n; ++i)
        if (j >= w.out0[i]) s = i;
    const int r = w.start[s] + w.lo[s] + (j - w.out0[s]);
    const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)r * d);
    uint4* dst = reinterpret_cast<uint4*>(xc + (size_t)j * d);
    for (int i = threadIdx.x; i < d / 8; i += blockDim.x) dst[i] = src[i];
}

int window_gather(const WinTable& w, const bf16* x, bf16* xc, int d, cudaStream_t stream) {
    const int Mw = w.out0[w.n];
    LaunchScope ls(LK_ROW, 2.0 * Mw * (double)d * 2, stream);
    MMDP_CUDA(launch_ex(window_gather_kernel, dim3(Mw), dim3(128), 0, stream, pdl_mode() != 0, false, w, x, xc, d));
    return 0;
}

// Packed row -> compact row of the head's requested rows: out[i] = the compact row of packed row rows[i]. A row outside the
// packed batch raises bit 1 of *err, a row outside its sequence's window bit 2 (the "row outside the window" flag of
// mmdp_model_forward_window); both then read compact row 0.
__global__ void window_row_map_kernel(const __grid_constant__ WinTable w, const int32_t* __restrict__ rows, int n,
                                      int32_t* __restrict__ out, int* __restrict__ err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = rows[i];
    int c = 0;
    if (r < 0 || r >= w.start[w.n]) {
        atomicOr(err, 2);
    } else {
        int s = 0;
        for (int k = 1; k < w.n; ++k)
            if (r >= w.start[k]) s = k;
        const int p = r - w.start[s];
        if (p < w.lo[s] || p >= w.hi[s]) atomicOr(err, 4);
        else c = w.out0[s] + p - w.lo[s];
    }
    out[i] = c;
}

int window_row_map(const WinTable& w, const int32_t* rows, int n, int32_t* out, int* err, cudaStream_t stream) {
    if (n <= 0) return 0;
    LaunchScope ls(LK_ROW, 8.0 * n, stream);
    window_row_map_kernel<<<(n + 255) / 256, 256, 0, stream>>>(w, rows, n, out, err);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int lfq_decode(const int64_t* ids, float* zq, int B, int N, int bits, cudaStream_t stream) {
    if (B <= 0 || N <= 0) return 0;
    if (bits <= 0 || bits > 62) return set_error("lfq_decode: bits out of range");
    dim3 grid((N + 255) / 256, B);
    LaunchScope ls(LK_ROW, (double)B * N * (8 + 4.0 * bits), stream);
    lfq_kernel<<<grid, 256, 0, stream>>>(ids, zq, N, bits);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace mmdp

struct LayerWeights {
    bf16* wqkv;       // [d + 2 d_kv, d]   rows: q_proj | k_proj | v_proj (d_kv = 128 n_kv_heads; d in a multi-head context)
    bf16* wo;         // [d, d]
    bf16* w13;        // [2ff, d]  128-row blocks interleaved: ff_proj block t, up_proj block t
    bf16* w2;         // [d, ff]
    bf16* attn_norm;  // [d]
    bf16* ff_norm;    // [d]
    // FP8 context: the four linears as e4m3 (same row order, except that W13 interleaves 64-row blocks, the gate / up halves
    // of the FP8 GEMM's 128-wide tile) with one fp32 scale per row; the bf16 pointers above are then null
    uint8_t *wqkv8 = nullptr, *wo8 = nullptr, *w13_8 = nullptr, *w2_8 = nullptr;
    float *sqkv = nullptr, *so = nullptr, *s13 = nullptr, *s2 = nullptr;
    bf16* qkv_bias = nullptr;  // MMDP_ARCH_QKV_BIAS: [d + 2 d_kv], q_bias | k_bias | v_bias
};

struct mmdp_model {
    mmdp_model_config cfg;
    // attention layout (mmdp_model_create_arch): kv heads and MMDP_ARCH_* flags. A context with n_kv_heads < n_heads or a bias
    // runs the grouped-query QKV epilogues; a plain multi-head one keeps EPI_QKVROPE(_PACKED)
    int n_kv_heads = 0, flags = 0;
    int d_kv() const { return n_kv_heads * 128; }
    bool gqa() const { return n_kv_heads != cfg.n_heads || flags != 0; }
    std::vector<LayerWeights> layers;
    bf16* wte = nullptr;
    bf16* ln_f = nullptr;
    bf16* head = nullptr;
    float* cos_tab = nullptr;
    float* sin_tab = nullptr;
    int rope_len = 0;
    // workspace
    int Mmax = 0, Lpad_max = 0;
    bf16 *x = nullptr, *xn = nullptr, *q = nullptr, *k = nullptr, *vt = nullptr, *att = nullptr, *h = nullptr, *xr = nullptr;
    int* err_flag = nullptr;  // device: bit 0 = token id out of range, bit 1 = logits row index out of range, bit 2 = row outside the window
    // V^T pad rule (vt_prepare): vt_Lpad = column stride of the layout the buffer was last zeroed for, vt_len[s] = columns
    // of block s written since then
    int vt_Lpad = 0;
    std::vector<int> vt_len;
    int2* seg_pos = nullptr;  // packed forward: (sequence, position) of every packed row
    int32_t* win_rows = nullptr;  // packed forward with row windows: the compact rows of the head's requested rows
    int precision = MMDP_PRECISION_BF16;
    uint8_t* a8 = nullptr;  // FP8: the quantised input of the current linear, [M, K] e4m3
    float* as = nullptr;    // FP8: its scales, [K / 128][M]
    std::vector<void*> allocs;
};

static int dev_alloc(mmdp_model* m, void** p, size_t bytes) {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) return set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    m->allocs.push_back(*p);
    return 0;
}

extern "C" {

MMDP_API int mmdp_version(void) { return MMDP_VERSION; }
MMDP_API const char* mmdp_last_error(void) { return last_error(); }

MMDP_API int mmdp_gemm_bf16(int epilogue, const uint16_t* A, int lda, const uint16_t* W, int ldw, int M, int N, int K,
                   uint16_t* C, int ldc, const uint16_t* R, int ldr, void* stream) {
    if (epilogue != MMDP_EPI_PLAIN && epilogue != MMDP_EPI_RESID && epilogue != MMDP_EPI_SWIGLU && epilogue != MMDP_EPI_F32)
        return set_error("mmdp_gemm_bf16: unknown epilogue %d", epilogue);
    return gemm_bf16(epilogue, (const bf16*)A, lda, (const bf16*)W, ldw, M, N, K, (bf16*)C, ldc, (const bf16*)R, ldr,
                     nullptr, (cudaStream_t)stream);
}

MMDP_API int mmdp_quantize_fp8(const uint16_t* x, int ldx, int rows, int K, int group, uint8_t* q, int ldq, float* scales, void* stream) {
    return quantize_fp8((const bf16*)x, ldx, rows, K, group, q, ldq, scales, (cudaStream_t)stream);
}

MMDP_API int mmdp_gemm_fp8(int epilogue, const uint8_t* A, int lda, const float* sa, const uint8_t* W, int ldw, const float* sw, int M,
                           int N, int K, uint16_t* C, int ldc, const uint16_t* R, int ldr, void* stream) {
    if (epilogue != MMDP_EPI_PLAIN && epilogue != MMDP_EPI_RESID && epilogue != MMDP_EPI_SWIGLU)
        return set_error("mmdp_gemm_fp8: unsupported epilogue %d", epilogue);
    return gemm_fp8(epilogue, A, lda, sa, W, ldw, sw, M, N, K, (bf16*)C, ldc, (const bf16*)R, ldr, nullptr, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads, int L, int Lpad,
                  const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_model, n_heads};
    return gemm_bf16(EPI_QKVROPE, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, 3 * d_model, d_model, nullptr, 0,
                     nullptr, 0, &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_gqa(const uint16_t* A, int lda, const uint16_t* Wqkv, const uint16_t* bias, int M, int d_model, int n_heads,
                               int n_kv_heads, int L, int Lpad, const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k,
                               uint16_t* vt, void* stream) {
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_model, n_heads};
    qa.n_kv_heads = n_kv_heads;
    qa.bias = (const bf16*)bias;
    return gemm_bf16(EPI_QKVGQA, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, d_model + 2 * 128 * n_kv_heads, d_model, nullptr, 0,
                     nullptr, 0, &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_tp(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads_local, int L,
                      int Lpad, const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    const int d_attn = n_heads_local * 128;
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_attn, n_heads_local};
    return gemm_bf16(EPI_QKVROPE, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, 3 * d_attn, d_model, nullptr, 0, nullptr, 0,
                     &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_tp_gqa(const uint16_t* A, int lda, const uint16_t* Wqkv, const uint16_t* bias, int M, int d_model,
                                  int n_heads_local, int n_kv_heads_local, int L, int Lpad, const float* cos_tab, const float* sin_tab,
                                  uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    const int d_attn = n_heads_local * 128;
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_attn, n_heads_local};
    qa.n_kv_heads = n_kv_heads_local;
    qa.bias = (const bf16*)bias;
    return gemm_bf16(EPI_QKVGQA, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, d_attn + 2 * 128 * n_kv_heads_local, d_model,
                     nullptr, 0, nullptr, 0, &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_tp_fp8(const uint8_t* A, int lda, const float* sa, const uint8_t* Wqkv, const float* sw, const uint16_t* bias,
                                  int M, int d_model, int n_heads_local, int n_kv_heads_local, int L, int Lpad, const float* cos_tab,
                                  const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    const int d_attn = n_heads_local * 128;
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_attn, n_heads_local};
    if (n_kv_heads_local == n_heads_local && !bias)
        return gemm_fp8(EPI_QKVROPE, A, lda, sa, Wqkv, d_model, sw, M, 3 * d_attn, d_model, nullptr, 0, nullptr, 0, &qa, (cudaStream_t)stream);
    qa.n_kv_heads = n_kv_heads_local;
    qa.bias = (const bf16*)bias;
    return gemm_fp8(EPI_QKVGQA, A, lda, sa, Wqkv, d_model, sw, M, d_attn + 2 * 128 * n_kv_heads_local, d_model, nullptr, 0, nullptr, 0,
                    &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_tp_packed(int precision, const void* A, int lda, const float* sa, const void* Wqkv, const float* sw,
                                     const uint16_t* bias, int d_model, int n_heads_local, int n_kv_heads_local, int n_seg,
                                     const int32_t* seg_len, int Lpad, const float* cos_tab, const float* sin_tab, uint16_t* q,
                                     uint16_t* k, uint16_t* vt, void* row_map, void* stream) {
    if (!A || !Wqkv || !row_map) return set_error("mmdp_qkv_rope_tp_packed: null argument");
    if (precision != MMDP_PRECISION_BF16 && precision != MMDP_PRECISION_FP8)
        return set_error("mmdp_qkv_rope_tp_packed: unknown precision %d", precision);
    if (precision == MMDP_PRECISION_FP8 && (!sa || !sw)) return set_error("mmdp_qkv_rope_tp_packed: FP8 needs the scales sa and sw");
    SegTable segs{};
    const int Lmax = seg_table("mmdp_qkv_rope_tp_packed", n_seg, seg_len, Lpad, &segs);
    if (Lmax < 0) return -1;
    if (Lpad % 8) return set_error("mmdp_qkv_rope_tp_packed: Lpad=%d must be a multiple of 8", Lpad);
    if (n_heads_local <= 0 || n_kv_heads_local <= 0 || n_heads_local % n_kv_heads_local || d_model <= 0)
        return set_error("mmdp_qkv_rope_tp_packed: n_kv_heads_local=%d must divide n_heads_local=%d", n_kv_heads_local, n_heads_local);
    const int M = segs.start[n_seg], da = n_heads_local * 128;
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, Lmax, Lpad, da, n_heads_local};
    qa.seg_pos = (const int2*)row_map;
    int epi = EPI_QKVROPE_PACKED, N = 3 * da;
    if (n_kv_heads_local != n_heads_local || bias) {
        epi = EPI_QKVGQA_PACKED;
        N = da + 2 * 128 * n_kv_heads_local;
        qa.n_kv_heads = n_kv_heads_local;
        qa.bias = (const bf16*)bias;
    }
    if (packed_row_map(segs, (int2*)row_map, (cudaStream_t)stream)) return -1;
    if (precision == MMDP_PRECISION_FP8)
        return gemm_fp8(epi, (const uint8_t*)A, lda, sa, (const uint8_t*)Wqkv, d_model, sw, M, N, d_model, nullptr, 0, nullptr, 0, &qa,
                        (cudaStream_t)stream);
    return gemm_bf16(epi, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, N, d_model, nullptr, 0, nullptr, 0, &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_resid_add_f32(uint16_t* x, int ldx, const float* partial, int ldp, int M, int d, void* stream) {
    return resid_add_f32((bf16*)x, ldx, partial, ldp, M, d, (cudaStream_t)stream);
}

MMDP_API int mmdp_attention(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, int n_heads, int L,
                   int Lpad, float scale, void* stream) {
    return attention_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, B, n_heads, L, Lpad, scale,
                         (cudaStream_t)stream);
}

MMDP_API int mmdp_attention_packed(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int n_seg, const int32_t* seg_len,
                                   int n_heads, int Lpad, float scale, void* stream) {
    if (!seg_len || n_seg <= 0 || n_seg > kMaxSegs) return set_error("mmdp_attention_packed: %d sequences (1 to %d)", n_seg, kMaxSegs);
    SegTable segs{};
    segs.n = n_seg;
    for (int i = 0; i < n_seg; ++i) segs.start[i + 1] = segs.start[i] + seg_len[i];
    return attention_packed_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, segs, n_heads, Lpad, scale, (cudaStream_t)stream);
}

MMDP_API int mmdp_attention_packed_window(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int n_seg,
                                          const int32_t* seg_len, const int32_t* win_lo, const int32_t* win_hi, int n_heads,
                                          int n_kv_heads, int Lpad, float scale, void* stream) {
    if (!seg_len || !win_lo || !win_hi || n_seg <= 0 || n_seg > kMaxSegs)
        return set_error("mmdp_attention_packed_window: %d sequences (1 to %d) with lengths and windows", n_seg, kMaxSegs);
    SegTable segs{};
    segs.n = n_seg;
    for (int i = 0; i < n_seg; ++i) segs.start[i + 1] = segs.start[i] + seg_len[i];
    return attention_packed_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, segs, n_heads, Lpad, scale, (cudaStream_t)stream,
                                n_kv_heads, win_lo, win_hi);
}

MMDP_API int mmdp_attention_gqa(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, const int32_t* seg_len,
                                int n_heads, int n_kv_heads, int L, int Lpad, float scale, void* stream) {
    if (n_kv_heads <= 0) return set_error("mmdp_attention_gqa: n_kv_heads must be positive");
    if (!seg_len)
        return attention_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, B, n_heads, L, Lpad, scale, (cudaStream_t)stream, 0,
                             n_kv_heads);
    if (B <= 0 || B > kMaxSegs) return set_error("mmdp_attention_gqa: %d sequences (1 to %d)", B, kMaxSegs);
    SegTable segs{};
    segs.n = B;
    for (int i = 0; i < B; ++i) segs.start[i + 1] = segs.start[i] + seg_len[i];
    return attention_packed_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, segs, n_heads, Lpad, scale, (cudaStream_t)stream,
                                n_kv_heads);
}

MMDP_API int mmdp_rmsnorm(const uint16_t* x, int ldx, const int32_t* rows, const uint16_t* weight, uint16_t* y, int ldy, int M,
                 int d, float eps, void* stream) {
    return rmsnorm_rows((const bf16*)x, ldx, rows, (const bf16*)weight, (bf16*)y, ldy, M, d, eps, (cudaStream_t)stream);
}

MMDP_API int mmdp_embed(const int64_t* ids, const uint16_t* wte, uint16_t* x, int M, int d, int64_t vocab, void* stream) {
    return embed_rows(ids, (const bf16*)wte, (bf16*)x, M, d, vocab, (cudaStream_t)stream);
}

MMDP_API int mmdp_text_step(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int R, int V, float text_cfg,
                   const uint16_t* unoise, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
                   int k, int64_t* x0_ws, double* conf_ws, void* stream) {
    return text_step((const bf16*)cond, (const bf16*)uncond, ld, R, V, text_cfg, (const bf16*)unoise, ld_noise,
                     temperature, ids_text, mask_id, k, x0_ws, conf_ws, (cudaStream_t)stream);
}

MMDP_API int mmdp_text_step_gumbel64(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int R, int V, float text_cfg,
                            const double* unoise64, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
                            int k, int64_t* x0_ws, double* conf_ws, void* stream) {
    if (!unoise64) return set_error("mmdp_text_step_gumbel64: noise pointer is null");
    return text_step((const bf16*)cond, (const bf16*)uncond, ld, R, V, text_cfg, nullptr, ld_noise, temperature, ids_text, mask_id, k,
                     x0_ws, conf_ws, (cudaStream_t)stream, unoise64);
}

MMDP_API int mmdp_image_step_t2i(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int N, int C, float cfg,
                        const uint16_t* gumbel_u, float tau, const uint16_t* conf_u, float temperature, int keep_n,
                        int64_t* ids, const int32_t* pos, int64_t mask_id, int64_t vq_offset, int32_t* sampled_ws,
                        float* selp_ws, uint8_t* unknown_ws, uint8_t* masking_out, void* stream) {
    return image_step_t2i((const bf16*)cond, (const bf16*)uncond, ld, N, C, cfg, (const bf16*)gumbel_u, tau, (const bf16*)conf_u,
                          temperature, keep_n, ids, pos, mask_id, vq_offset, sampled_ws, selp_ws, unknown_ws, masking_out,
                          (cudaStream_t)stream);
}

MMDP_API int mmdp_image_step(int variant, const uint16_t* cond, const uint16_t* unc_a, const uint16_t* unc_b, int64_t ld, int N,
                    int C, float s_a, float s_b, const uint16_t* qnoise, const uint16_t* conf_noise, float temp,
                    int sched_len, int64_t* ids, const int32_t* pos, int64_t mask_id, int64_t vq_offset,
                    int32_t* sampled_ws, float* selp_ws, uint8_t* unknown_ws, uint16_t* probs_out,
                    int32_t* mask_len_out, uint8_t* masking_out, void* stream) {
    if (variant != 0 && variant != 1) return set_error("mmdp_image_step: variant must be 0 (A) or 1 (M)");
    return image_step(variant, (const bf16*)cond, (const bf16*)unc_a, (const bf16*)unc_b, ld, N, C, s_a, s_b,
                      (const bf16*)qnoise, (const bf16*)conf_noise, temp, sched_len, ids, pos, mask_id, vq_offset,
                      sampled_ws, selp_ws, unknown_ws, (bf16*)probs_out, mask_len_out, masking_out,
                      (cudaStream_t)stream);
}

MMDP_API int mmdp_image_remask(int variant, int N, const int32_t* sampled, const float* selp, const uint8_t* unknown,
                      const uint16_t* conf_noise, float temp, int sched_len, int64_t* ids, const int32_t* pos,
                      int64_t mask_id, int64_t vq_offset, int32_t* mask_len_out, uint8_t* masking_out, void* stream) {
    if (variant != 0 && variant != 1) return set_error("mmdp_image_remask: variant must be 0 (A) or 1 (M)");
    return image_remask(variant, N, sampled, selp, unknown, (const bf16*)conf_noise, temp, sched_len, ids, pos, mask_id,
                        vq_offset, mask_len_out, masking_out, (cudaStream_t)stream);
}

MMDP_API int mmdp_lfq_decode(const int64_t* ids, float* zq, int B, int N, int bits, void* stream) {
    return lfq_decode(ids, zq, B, N, bits, (cudaStream_t)stream);
}

// ---- tensor-parallel plumbing: device buffers shared between the ranks of one node through CUDA IPC ------------------------
MMDP_API int mmdp_tp_alloc(uint64_t bytes, void** out) {
    if (!out || bytes == 0) return set_error("mmdp_tp_alloc: bad arguments");
    MMDP_CUDA(cudaMalloc(out, bytes));
    MMDP_CUDA(cudaMemset(*out, 0, bytes));
    return 0;
}
MMDP_API int mmdp_tp_free(void* p) {
    if (p) MMDP_CUDA(cudaFree(p));
    return 0;
}
MMDP_API int mmdp_ipc_export(void* p, uint8_t* handle64) {
    if (!p || !handle64) return set_error("mmdp_ipc_export: null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    MMDP_CUDA(cudaIpcGetMemHandle(&h, p));
    memcpy(handle64, &h, 64);
    return 0;
}
MMDP_API int mmdp_ipc_import(const uint8_t* handle64, void** out) {
    if (!handle64 || !out) return set_error("mmdp_ipc_import: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    MMDP_CUDA(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));  // maps the peer's buffer; enables P2P access
    return 0;
}
MMDP_API int mmdp_ipc_close(void* p) {
    if (p) MMDP_CUDA(cudaIpcCloseMemHandle(p));
    return 0;
}
MMDP_API int mmdp_tp_reduce_norm(const float* recv_local, int rows_per_rank, int n_src, uint16_t* const* xn, uint32_t* const* flags,
                        int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* weight, int row0, int nrows, int d, float eps,
                        uint32_t epoch, uint32_t* done_counter, void* stream) {
    return tp_reduce_norm(recv_local, rows_per_rank, n_src, xn, flags, n_ranks, my_rank, x_shard, weight, row0, nrows, d, eps, epoch,
                          done_counter, (cudaStream_t)stream);
}
MMDP_API int mmdp_gemm_f32_scatter(const uint16_t* A, int lda, const uint16_t* W, int ldw, int M, int N, int K, float* const* recv,
                          int n_ranks, int rows_per_rank, int slot, void* stream) {
    if (!recv || n_ranks < 1 || n_ranks > 8) return set_error("mmdp_gemm_f32_scatter: bad rank layout");
    // the receive buffers hold n_ranks slots: a slot past them would be pushed beyond the owner's buffer
    if (slot < 0 || slot >= n_ranks) return set_error("mmdp_gemm_f32_scatter: slot %d outside [0, %d)", slot, n_ranks);
    if (rows_per_rank <= 0 || (M + rows_per_rank - 1) / rows_per_rank > n_ranks) return set_error("mmdp_gemm_f32_scatter: M does not fit n_ranks x rows_per_rank");
    GemmScatter sc{};
    for (int r = 0; r < n_ranks; ++r) sc.dst[r] = recv[r];
    sc.rows_per_rank = rows_per_rank; sc.slot = slot;
    return gemm_bf16(EPI_F32, (const bf16*)A, lda, (const bf16*)W, ldw, M, N, K, nullptr, N, nullptr, 0, nullptr, (cudaStream_t)stream, &sc);
}

MMDP_API int mmdp_gemm_fp8_f32(const uint8_t* A, int lda, const float* sa, const uint8_t* W, int ldw, const float* sw, int M, int N, int K,
                               float* C, int ldc, void* stream) {
    if (!C) return set_error("mmdp_gemm_fp8_f32: C is null");
    return gemm_fp8(EPI_F32, A, lda, sa, W, ldw, sw, M, N, K, (bf16*)C, ldc, nullptr, 0, nullptr, (cudaStream_t)stream);
}
MMDP_API int mmdp_gemm_fp8_f32_scatter(const uint8_t* A, int lda, const float* sa, const uint8_t* W, int ldw, const float* sw, int M, int N,
                                       int K, float* const* recv, int n_ranks, int rows_per_rank, int slot, void* stream) {
    if (!recv || n_ranks < 1 || n_ranks > 8) return set_error("mmdp_gemm_fp8_f32_scatter: bad rank layout");
    if (slot < 0 || slot >= n_ranks) return set_error("mmdp_gemm_fp8_f32_scatter: slot %d outside [0, %d)", slot, n_ranks);
    if (rows_per_rank <= 0 || (M + rows_per_rank - 1) / rows_per_rank > n_ranks)
        return set_error("mmdp_gemm_fp8_f32_scatter: M does not fit n_ranks x rows_per_rank");
    GemmScatter sc{};
    for (int r = 0; r < n_ranks; ++r) sc.dst[r] = recv[r];
    sc.rows_per_rank = rows_per_rank; sc.slot = slot;
    return gemm_fp8(EPI_F32, A, lda, sa, W, ldw, sw, M, N, K, nullptr, N, nullptr, 0, nullptr, (cudaStream_t)stream, &sc);
}
MMDP_API int mmdp_tp_reduce_norm_fp8(const float* recv_local, int rows_per_rank, int n_src, uint8_t* const* xq, float* const* xs, int ld_s,
                                     uint32_t* const* flags, int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* weight, int row0,
                                     int nrows, int d, float eps, uint32_t epoch, uint32_t* done_counter, void* stream) {
    return tp_reduce_norm_fp8(recv_local, rows_per_rank, n_src, xq, xs, ld_s, flags, n_ranks, my_rank, x_shard, weight, row0, nrows, d, eps,
                              epoch, done_counter, (cudaStream_t)stream);
}

// second stream + events of the two-chunk tensor-parallel forward, one set per device
struct TpSide { cudaStream_t s1 = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };
static int tp_side(TpSide** out) {
    static TpSide sides[64];
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    TpSide& t = sides[dev & 63];
    if (!t.s1) {
        MMDP_CUDA(cudaStreamCreateWithFlags(&t.s1, cudaStreamNonBlocking));
        MMDP_CUDA(cudaEventCreateWithFlags(&t.fork, cudaEventDisableTiming));
        MMDP_CUDA(cudaEventCreateWithFlags(&t.join, cudaEventDisableTiming));
    }
    *out = &t;
    return 0;
}

// The tensor-parallel body of mmdp_tp_forward (segs == nullptr: B sequences of L rows) and mmdp_tp_forward_packed (segs: the
// packed batch, whose sizes the caller has checked; L = the longest sequence). Only the QKV epilogue, the attention launch and the
// V^T layout see the sequences; everything else works on the M rows.
static int tp_forward(const mmdp_tp_ctx* c, const int64_t* ids, const SegTable* segs, int B, int L, uint32_t epoch0, uint32_t* epoch_out,
                      void* stream) {
    cudaStream_t s0 = (cudaStream_t)stream;
    const int d = c->d_model, Hl = c->n_heads_local, da = Hl * 128, ffl = c->ff_local, tp = c->n_ranks;
    // kv heads of this rank's shard: 0 = Hl (the multi-head shard)
    const int Hkv = c->n_kv_heads_local ? c->n_kv_heads_local : Hl, dkv = Hkv * 128;
    if (Hkv <= 0 || Hkv > Hl || Hl % Hkv)
        return set_error("mmdp_tp_forward: n_kv_heads_local=%d must divide n_heads_local=%d", c->n_kv_heads_local, Hl);
    const int M = segs ? segs->start[segs->n] : B * L, Lpad = ((L + 7) / 8) * 8;
    const int2* seg_pos = segs ? (const int2*)c->packed.seg_pos : nullptr;
    const int nch = c->n_chunks == 2 ? 2 : 1;
    if (c->precision != MMDP_PRECISION_BF16 && c->precision != MMDP_PRECISION_FP8)
        return set_error("mmdp_tp_forward: unknown precision %d", c->precision);
    const bool f8 = c->precision == MMDP_PRECISION_FP8;
    if (f8 && (!c->layers_fp8 || !c->xq || !c->xq_scales || !c->a8 || !c->a8_scales))
        return set_error("mmdp_tp_forward: an FP8 context needs layers_fp8, xq, xq_scales, a8 and a8_scales");
    if (f8 && (d % 128 || ffl % 128)) return set_error("mmdp_tp_forward: FP8 needs d_model and ff_local multiples of 128");
    const int ka = da > ffl ? da : ffl;  // FP8: row stride of a chunk's region of a8 (att and h of a chunk share it)
    if (nch == 2 && (c->chunk_rows0 <= 0 || c->chunk_rows0 >= M)) return set_error("mmdp_tp_forward: chunk_rows0 must lie inside (0, %d)", M);
    // row chunks: chunk ci covers sequence rows [m0, m0 + Mc); inside it rank r owns [r * R, (r + 1) * R)
    struct Chunk { int m0, Mc, R, row0, nrows; cudaStream_t s; GemmScatter sc[2]; };
    Chunk ch[2];
    TpSide* side = nullptr;
    if (nch == 2 && tp_side(&side)) return -1;
    for (int ci = 0; ci < nch; ++ci) {
        Chunk& k = ch[ci];
        k.m0 = ci == 0 ? 0 : c->chunk_rows0;
        k.Mc = nch == 1 ? M : (ci == 0 ? c->chunk_rows0 : M - c->chunk_rows0);
        k.R = (k.Mc + tp - 1) / tp;
        k.row0 = c->rank * k.R;
        k.nrows = k.Mc - k.row0 < k.R ? k.Mc - k.row0 : k.R;
        if (k.nrows < 1 || k.Mc - (tp - 1) * k.R < 1)
            return set_error("mmdp_tp_forward: %d rows cannot be split over %d ranks with at least one row each", k.Mc, tp);
    }
    for (int ci = 0; ci < nch; ++ci) {  // the chunks' shared buffers are read only once every chunk's split is checked
        Chunk& k = ch[ci];
        k.s = ci == 0 ? s0 : side->s1;
        for (int b = 0; b < 2; ++b) {
            k.sc[b] = GemmScatter{};
            for (int r = 0; r < tp; ++r) k.sc[b].dst[r] = c->chunk[ci].recv[b][r];
            k.sc[b].rows_per_rank = k.R; k.sc[b].slot = c->rank;
        }
    }
    const float scale = 1.0f / sqrtf(128.0f);
    uint32_t epoch = epoch0;
    // this rank's view of every rank's activation buffer, offset to the chunk's first row
    uint16_t* xn_chunk[2][8];
    // FP8: the same views of the e4m3 activation buffers; chunk ci's scales are a [d / 128][Mc] block at m0 * d / 128
    uint8_t* xq_chunk[2][8];
    float* xs_chunk[2][8];
    for (int ci = 0; ci < nch; ++ci)
        for (int r = 0; r < tp; ++r) {
            xn_chunk[ci][r] = c->xn[r] + (size_t)ch[ci].m0 * d;
            xq_chunk[ci][r] = f8 ? c->xq[r] + (size_t)ch[ci].m0 * d : nullptr;
            xs_chunk[ci][r] = f8 ? c->xq_scales[r] + (size_t)ch[ci].m0 * (d / 128) : nullptr;
        }
    // the reduce before a column-parallel linear broadcasts e4m3 in FP8; the last one (ln_f, read by the bf16 LM head) bf16
    auto reduce = [&](int ci, int buf, const uint16_t* w, uint32_t ep, bool to_fp8) -> int {
        const Chunk& k = ch[ci];
        const mmdp_tp_chunk& cc = c->chunk[ci];
        const float* recv = buf >= 0 ? cc.recv[buf][c->rank] : nullptr;
        if (to_fp8)
            return tp_reduce_norm_fp8(recv, k.R, buf >= 0 ? tp : 0, xq_chunk[ci], xs_chunk[ci], k.Mc, cc.flags, tp, c->rank, cc.x_shard, w,
                                      k.row0, k.nrows, d, c->rms_eps, ep, cc.done_counter, k.s);
        return tp_reduce_norm(recv, k.R, buf >= 0 ? tp : 0, xn_chunk[ci], cc.flags, tp, c->rank, cc.x_shard, w,
                              k.row0, k.nrows, d, c->rms_eps, ep, cc.done_counter, k.s);
    };
    // FP8: chunk ci's local e4m3 copy of att / h (K columns) and its scales, a region of a8 no other chunk touches
    auto quant_local = [&](int ci, const bf16* x, int K, uint8_t** q, float** sq) -> int {
        const Chunk& k = ch[ci];
        *q = c->a8 + (size_t)k.m0 * ka;
        *sq = c->a8_scales + (size_t)k.m0 * (ka / 128);
        return quantize_fp8(x, K, k.Mc, K, 128, *q, K, *sq, k.s);
    };
    auto fork = [&]() -> int {  // the side stream continues after everything issued to the caller's stream so far
        if (nch == 1) return 0;
        MMDP_CUDA(cudaEventRecord(side->fork, s0));
        MMDP_CUDA(cudaStreamWaitEvent(side->s1, side->fork, 0));
        return 0;
    };
    auto join = [&]() -> int {
        if (nch == 1) return 0;
        MMDP_CUDA(cudaEventRecord(side->join, side->s1));
        MMDP_CUDA(cudaStreamWaitEvent(s0, side->join, 0));
        return 0;
    };
    const bf16* xn = (const bf16*)c->xn[c->rank];
    if (segs && packed_row_map(*segs, (int2*)c->packed.seg_pos, s0)) return -1;
    if (fork()) return -1;
    ++epoch;
    for (int ci = 0; ci < nch; ++ci) {
        const Chunk& k = ch[ci];
        if (embed_rows(ids + k.m0 + k.row0, (const bf16*)c->wte, (bf16*)c->chunk[ci].x_shard, k.nrows, d, c->vocab, k.s, nullptr)) return -1;
        if (reduce(ci, -1, c->layers[0].attn_norm, epoch, f8)) return -1;
    }
    for (int li = 0; li < c->n_layers; ++li) {
        const mmdp_tp_layer& l = c->layers[li];
        const mmdp_tp_layer_fp8* l8 = f8 ? &c->layers_fp8[li] : nullptr;
        // a grouped-query or biased shard runs the grouped-query epilogue; the multi-head shard keeps EPI_QKVROPE
        const bool gqa = Hkv != Hl || l.bqkv;
        for (int ci = 0; ci < nch; ++ci) {
            const Chunk& k = ch[ci];
            QkvRopeArgs qa{(bf16*)c->q + (size_t)k.m0 * da, (bf16*)c->k + (size_t)k.m0 * dkv, (bf16*)c->vt, c->cos_tab, c->sin_tab, L, Lpad, da, Hl};
            // packed: chunk ci's GEMM row r is packed row m0 + r, so it reads the row map from m0 as q / k start at m0
            if (segs) qa.seg_pos = seg_pos + k.m0;
            else { qa.chunked = nch > 1; qa.row0 = k.m0; }
            if (gqa) { qa.n_kv_heads = Hkv; qa.bias = (const bf16*)l.bqkv; }
            const int epi = segs ? (gqa ? EPI_QKVGQA_PACKED : EPI_QKVROPE_PACKED) : (gqa ? EPI_QKVGQA : EPI_QKVROPE);
            if (f8 ? gemm_fp8(epi, xq_chunk[ci][c->rank], d, xs_chunk[ci][c->rank], l8->wqkv, d, l8->sqkv, k.Mc, da + 2 * dkv, d, nullptr, 0,
                              nullptr, 0, &qa, k.s)
                   : gemm_bf16(epi, xn + (size_t)k.m0 * d, d, (const bf16*)l.wqkv, d, k.Mc, da + 2 * dkv, d, nullptr, 0, nullptr, 0, &qa, k.s))
                return -1;
        }
        // attention mixes all rows: both chunks' q / k / v^T must be complete, and it must be complete before either chain goes on
        if (join()) return -1;
        if (segs ? attention_packed_fwd((const bf16*)c->q, (const bf16*)c->k, (const bf16*)c->vt, (bf16*)c->att, *segs, Hl, Lpad, scale, s0, Hkv)
                 : attention_fwd((const bf16*)c->q, (const bf16*)c->k, (const bf16*)c->vt, (bf16*)c->att, B, Hl, L, Lpad, scale, s0, 0, Hkv))
            return -1;
        if (fork()) return -1;
        const uint32_t e1 = ++epoch, e2 = ++epoch;
        for (int ci = 0; ci < nch; ++ci) {
            const Chunk& k = ch[ci];
            const bf16* att = (const bf16*)c->att + (size_t)k.m0 * da;
            bf16* h = (bf16*)c->h + (size_t)k.m0 * ffl;
            const bool last = li + 1 == c->n_layers;
            if (f8) {
                uint8_t* q8;
                float* s8;
                if (quant_local(ci, att, da, &q8, &s8)) return -1;
                if (gemm_fp8(EPI_F32, q8, da, s8, l8->wo, da, l8->so, k.Mc, d, da, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[0])) return -1;
                if (reduce(ci, 0, l.ff_norm, e1, true)) return -1;
                if (gemm_fp8(EPI_SWIGLU, xq_chunk[ci][c->rank], d, xs_chunk[ci][c->rank], l8->w13, d, l8->s13, k.Mc, 2 * ffl, d, h, ffl, nullptr,
                             0, nullptr, k.s))
                    return -1;
                if (quant_local(ci, h, ffl, &q8, &s8)) return -1;
                if (gemm_fp8(EPI_F32, q8, ffl, s8, l8->w2, ffl, l8->s2, k.Mc, d, ffl, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[1])) return -1;
            } else {
                if (gemm_bf16(EPI_F32, att, da, (const bf16*)l.wo, da, k.Mc, d, da, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[0])) return -1;
                if (reduce(ci, 0, l.ff_norm, e1, false)) return -1;
                if (gemm_bf16(EPI_SWIGLU, xn + (size_t)k.m0 * d, d, (const bf16*)l.w13, d, k.Mc, 2 * ffl, d, h, ffl, nullptr, 0, nullptr, k.s)) return -1;
                if (gemm_bf16(EPI_F32, h, ffl, (const bf16*)l.w2, ffl, k.Mc, d, ffl, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[1])) return -1;
            }
            if (reduce(ci, 1, last ? c->ln_f : c->layers[li + 1].attn_norm, e2, f8 && !last)) return -1;
        }
    }
    if (join()) return -1;
    *epoch_out = epoch;
    return 0;
}

MMDP_API int mmdp_tp_forward(const mmdp_tp_ctx* c, const int64_t* ids, int B, int L, uint32_t epoch0, uint32_t* epoch_out, void* stream) {
    if (!c || !ids || !epoch_out) return set_error("mmdp_tp_forward: null argument");
    return tp_forward(c, ids, nullptr, B, L, epoch0, epoch_out, stream);
}

MMDP_API int mmdp_tp_forward_packed(const mmdp_tp_ctx* c, const int64_t* ids, int n_seg, const int32_t* seg_len, uint32_t epoch0,
                                    uint32_t* epoch_out, void* stream) {
    if (!c || !ids || !epoch_out) return set_error("mmdp_tp_forward_packed: null argument");
    if (!c->packed.seg_pos || c->packed.max_rows <= 0 || c->packed.rope_len <= 0)
        return set_error("mmdp_tp_forward_packed: the context has no packed row map (packed.seg_pos, max_rows, rope_len)");
    SegTable segs{};
    const int Lmax = seg_table("mmdp_tp_forward_packed", n_seg, seg_len, c->packed.rope_len, &segs);
    if (Lmax < 0) return -1;
    if (segs.start[n_seg] > c->packed.max_rows)
        return set_error("mmdp_tp_forward_packed: %d packed rows exceed the workspace of %d", segs.start[n_seg], c->packed.max_rows);
    return tp_forward(c, ids, &segs, n_seg, Lmax, epoch0, epoch_out, stream);
}

MMDP_API void mmdp_prof_enable(int on) { prof_enable(on); }
MMDP_API int mmdp_prof_summary(double* ms, double* work, long long* launches) { return prof_summary(ms, work, launches); }
MMDP_API void mmdp_set_gemm_pair(int on) { set_gemm_pair_mode(on); }
MMDP_API long long mmdp_launch_count(int reset) { return launch_count(reset); }
MMDP_API void mmdp_set_gemm_splitk(int mode) { set_gemm_splitk_mode(mode < 0 ? 0 : (mode > 3 ? 3 : mode)); }
MMDP_API void mmdp_set_pdl(int on) { set_pdl_mode(on); }
MMDP_API int mmdp_set_option(const char* key, int value) { return key ? set_opt(key, value) : set_error("mmdp_set_option: null key"); }

// ------------------------------------------------------------------------------------------------
// model context
// ------------------------------------------------------------------------------------------------
MMDP_API int mmdp_model_create(const mmdp_model_config* c, mmdp_model** out) {
    return mmdp_model_create_ex(c, MMDP_PRECISION_BF16, out);
}

MMDP_API int mmdp_model_create_ex(const mmdp_model_config* c, int precision, mmdp_model** out) {
    if (!c) return set_error("mmdp_model_create: null argument");
    return mmdp_model_create_arch(c, precision, c->n_heads, 0, out);
}

MMDP_API int mmdp_model_create_arch(const mmdp_model_config* c, int precision, int n_kv_heads, int flags, mmdp_model** out) {
    if (!c || !out) return set_error("mmdp_model_create: null argument");
    if (n_kv_heads <= 0 || n_kv_heads > c->n_heads || c->n_heads % n_kv_heads)
        return set_error("mmdp_model_create: n_kv_heads=%d must divide n_heads=%d", n_kv_heads, c->n_heads);
    if (flags & ~MMDP_ARCH_QKV_BIAS) return set_error("mmdp_model_create: unknown architecture flags 0x%x", flags);
    if (precision != MMDP_PRECISION_BF16 && precision != MMDP_PRECISION_FP8)
        return set_error("mmdp_model_create: unknown precision %d", precision);
    if (c->d_model != c->n_heads * 128) return set_error("mmdp_model_create: head_dim must be 128");
    if (c->d_model % 256) return set_error("mmdp_model_create: d_model must be a multiple of 256");
    // (both also make every K of the FP8 linears a multiple of its 128-wide activation scale group)
    if (c->mlp_hidden % 128) return set_error("mmdp_model_create: mlp_hidden must be a multiple of 128");
    if (c->vocab_size % 8) return set_error("mmdp_model_create: vocab_size must be a multiple of 8");
    if (c->n_layers <= 0 || c->max_seq_len <= 0 || c->max_batch <= 0) return set_error("mmdp_model_create: bad sizes");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return set_error("mmdp_model_create: no CUDA device (this library has no CPU fallback)");
    mmdp_model* m = new mmdp_model();
    m->cfg = *c;
    m->precision = precision;
    m->n_kv_heads = n_kv_heads;
    m->flags = flags;
    const size_t d = c->d_model, ff = c->mlp_hidden, V = c->vocab_size, dkv = m->d_kv(), nqkv = d + 2 * dkv;
    m->layers.resize(c->n_layers);
    int rc = 0;
    for (auto& l : m->layers) {
        if (flags & MMDP_ARCH_QKV_BIAS) rc |= dev_alloc(m, (void**)&l.qkv_bias, nqkv * 2);
        if (precision == MMDP_PRECISION_FP8) {
            rc |= dev_alloc(m, (void**)&l.wqkv8, nqkv * d);
            rc |= dev_alloc(m, (void**)&l.wo8, d * d);
            rc |= dev_alloc(m, (void**)&l.w13_8, 2 * ff * d);
            rc |= dev_alloc(m, (void**)&l.w2_8, d * ff);
            rc |= dev_alloc(m, (void**)&l.sqkv, nqkv * 4);
            rc |= dev_alloc(m, (void**)&l.so, d * 4);
            rc |= dev_alloc(m, (void**)&l.s13, 2 * ff * 4);
            rc |= dev_alloc(m, (void**)&l.s2, d * 4);
        } else {
            rc |= dev_alloc(m, (void**)&l.wqkv, nqkv * d * 2);
            rc |= dev_alloc(m, (void**)&l.wo, d * d * 2);
            rc |= dev_alloc(m, (void**)&l.w13, 2 * ff * d * 2);
            rc |= dev_alloc(m, (void**)&l.w2, d * ff * 2);
        }
        rc |= dev_alloc(m, (void**)&l.attn_norm, d * 2);
        rc |= dev_alloc(m, (void**)&l.ff_norm, d * 2);
    }
    rc |= dev_alloc(m, (void**)&m->wte, V * d * 2);
    rc |= dev_alloc(m, (void**)&m->head, V * d * 2);
    rc |= dev_alloc(m, (void**)&m->ln_f, d * 2);
    m->Mmax = c->max_batch * c->max_seq_len;
    m->Lpad_max = ((c->max_seq_len + 127) / 128) * 128;
    const size_t Mm = m->Mmax;
    rc |= dev_alloc(m, (void**)&m->x, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->xn, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->q, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->k, Mm * dkv * 2);
    rc |= dev_alloc(m, (void**)&m->att, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->xr, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->h, Mm * ff * 2);
    if (precision == MMDP_PRECISION_FP8) {  // the widest linear input is h: K = mlp_hidden
        rc |= dev_alloc(m, (void**)&m->a8, Mm * ff);
        rc |= dev_alloc(m, (void**)&m->as, Mm * (ff / 128) * 4);
    }
    rc |= dev_alloc(m, (void**)&m->vt, (size_t)c->max_batch * dkv * m->Lpad_max * 2);
    rc |= dev_alloc(m, (void**)&m->cos_tab, (size_t)c->max_seq_len * 64 * 4);
    rc |= dev_alloc(m, (void**)&m->sin_tab, (size_t)c->max_seq_len * 64 * 4);
    rc |= dev_alloc(m, (void**)&m->err_flag, sizeof(int));
    rc |= dev_alloc(m, (void**)&m->seg_pos, Mm * sizeof(int2));
    rc |= dev_alloc(m, (void**)&m->win_rows, Mm * sizeof(int32_t));
    m->vt_len.assign(c->max_batch, 0);
    if (!rc && cudaMemset(m->err_flag, 0, sizeof(int)) != cudaSuccess) rc = set_error("mmdp_model_create: cudaMemset failed");
    if (rc) {
        mmdp_model_destroy(m);
        return -1;
    }
    *out = m;
    return 0;
}

MMDP_API void mmdp_model_destroy(mmdp_model* m) {
    if (!m) return;
    for (void* p : m->allocs) cudaFree(p);
    delete m;
}

static int copy_rows(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    MMDP_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
    return 0;
}

// FP8 context: one linear of a block [rows, cols] (bf16, device or host) -> e4m3 with one scale per row (group = cols), written
// into the packed layer matrices. The bf16 source is staged on the device and never kept.
// qkv_row0: first row of q_proj / k_proj / v_proj inside the packed Wqkv (0, d, d + d_kv)
static int set_weight_fp8(LayerWeights& l, const char* sub, const void* src, int64_t rows, int64_t cols, int64_t qkv_row0, cudaStream_t s) {
    const size_t n = (size_t)rows * cols;
    const bool w13 = !strcmp(sub, "up_proj") || !strcmp(sub, "ff_proj");
    bf16* stage = nullptr;
    uint8_t* q = nullptr;
    float* sc = nullptr;
    MMDP_CUDA(cudaMallocAsync((void**)&stage, n * 2 + (w13 ? n + rows * 4 : 0), s));
    int rc = copy_rows(stage, src, n * 2, s);
    if (!strcmp(sub, "attn_out")) { q = l.wo8; sc = l.so; }
    else if (!strcmp(sub, "ff_out")) { q = l.w2_8; sc = l.s2; }
    else if (!w13) {
        q = l.wqkv8 + (size_t)qkv_row0 * cols;
        sc = l.sqkv + qkv_row0;
    } else {  // quantised next to the stage, then interleaved: source block t of 64 rows -> destination block 2t + up
        q = reinterpret_cast<uint8_t*>(stage + n);
        sc = reinterpret_cast<float*>(q + n);
    }
    if (!rc) rc = quantize_fp8(stage, (int)cols, (int)rows, (int)cols, (int)cols, q, (int)cols, sc, s);
    if (!rc && w13) {
        const size_t up = !strcmp(sub, "up_proj") ? 1 : 0;
        const cudaError_t e1 = cudaMemcpy2DAsync(l.w13_8 + up * 64 * cols, 128 * cols, q, 64 * cols, 64 * cols, rows / 64,
                                                 cudaMemcpyDeviceToDevice, s);
        const cudaError_t e2 = cudaMemcpy2DAsync(l.s13 + up * 64, 128 * 4, sc, 64 * 4, 64 * 4, rows / 64, cudaMemcpyDeviceToDevice, s);
        if (e1 != cudaSuccess || e2 != cudaSuccess) rc = set_error("mmdp_model_set_weight: packing W13 failed: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
    }
    const cudaError_t ef = cudaFreeAsync(stage, s);
    if (!rc && ef != cudaSuccess) rc = set_error("mmdp_model_set_weight: cudaFreeAsync failed: %s", cudaGetErrorString(ef));
    return rc;
}

MMDP_API int mmdp_model_set_weight(mmdp_model* m, const char* name, const void* src, int64_t rows, int64_t cols, void* stream) {
    if (!m || !name || !src) return set_error("mmdp_model_set_weight: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t d = m->cfg.d_model, ff = m->cfg.mlp_hidden, V = m->cfg.vocab_size, dkv = m->d_kv();
    auto expect = [&](int64_t r, int64_t c) -> int {
        if (rows != r || cols != c)
            return set_error("mmdp_model_set_weight(%s): expected [%lld,%lld], got [%lld,%lld]", name, (long long)r,
                             (long long)c, (long long)rows, (long long)cols);
        return 0;
    };
    const uint8_t* sb = (const uint8_t*)src;
    if (!strcmp(name, "wte")) { if (expect(V, d)) return -1; return copy_rows(m->wte, src, V * d * 2, s); }
    if (!strcmp(name, "head")) { if (expect(V, d)) return -1; return copy_rows(m->head, src, V * d * 2, s); }
    if (!strcmp(name, "ln_f")) { if (expect(d, 1) && expect(1, d)) return -1; return copy_rows(m->ln_f, src, d * 2, s); }
    int li = -1;
    char sub[64];
    if (sscanf(name, "blocks.%d.%63s", &li, sub) != 2 || li < 0 || li >= m->cfg.n_layers)
        return set_error("mmdp_model_set_weight: unknown tensor name '%s'", name);
    LayerWeights& l = m->layers[li];
    // q_proj | k_proj | v_proj rows of the packed Wqkv (and of the bias): [0, d), [d, d + d_kv), [d + d_kv, d + 2 d_kv)
    const bool qkv = !strcmp(sub, "q_proj") || !strcmp(sub, "k_proj") || !strcmp(sub, "v_proj");
    const int64_t qkv_row0 = sub[0] == 'q' ? 0 : (sub[0] == 'k' ? d : d + dkv), qkv_rows = sub[0] == 'q' ? d : dkv;
    if (!strcmp(sub, "q_bias") || !strcmp(sub, "k_bias") || !strcmp(sub, "v_bias")) {
        if (!l.qkv_bias) return set_error("mmdp_model_set_weight(%s): the context was created without MMDP_ARCH_QKV_BIAS", name);
        if (expect(qkv_rows, 1) && expect(1, qkv_rows)) return -1;
        return copy_rows(l.qkv_bias + qkv_row0, src, qkv_rows * 2, s);
    }
    if (m->precision == MMDP_PRECISION_FP8) {
        const bool w13 = !strcmp(sub, "ff_proj") || !strcmp(sub, "up_proj");
        const bool wo = !strcmp(sub, "attn_out"), w2 = !strcmp(sub, "ff_out");
        if (qkv || w13 || wo || w2) {
            const int64_t r = w13 ? ff : (qkv ? qkv_rows : d), k = w2 ? ff : d;
            if (expect(r, k)) return -1;
            return set_weight_fp8(l, sub, src, r, k, qkv_row0, s);
        }
    }
    if (qkv) {
        if (expect(qkv_rows, d)) return -1;
        return copy_rows(l.wqkv + (size_t)qkv_row0 * d, src, qkv_rows * d * 2, s);
    }
    if (!strcmp(sub, "attn_out")) { if (expect(d, d)) return -1; return copy_rows(l.wo, src, d * d * 2, s); }
    if (!strcmp(sub, "ff_out")) { if (expect(d, ff)) return -1; return copy_rows(l.w2, src, d * ff * 2, s); }
    if (!strcmp(sub, "attn_norm")) { if (expect(d, 1) && expect(1, d)) return -1; return copy_rows(l.attn_norm, src, d * 2, s); }
    if (!strcmp(sub, "ff_norm")) { if (expect(d, 1) && expect(1, d)) return -1; return copy_rows(l.ff_norm, src, d * 2, s); }
    if (!strcmp(sub, "ff_proj") || !strcmp(sub, "up_proj")) {
        if (expect(ff, d)) return -1;
        const int up = sub[0] == 'u' ? 1 : 0;
        // one 2-D copy: source block t (128 rows, contiguous 128*d) -> destination block 2t+up
        MMDP_CUDA(cudaMemcpy2DAsync(l.w13 + (size_t)up * 128 * d, (size_t)256 * d * 2, sb, (size_t)128 * d * 2,
                                    (size_t)128 * d * 2, (size_t)(ff / 128), cudaMemcpyDefault, s));
        return 0;
    }
    return set_error("mmdp_model_set_weight: unknown tensor name '%s'", name);
}

MMDP_API int mmdp_model_set_rope(mmdp_model* m, const float* cos_tab, const float* sin_tab, int L, void* stream) {
    if (!m || !cos_tab || !sin_tab) return set_error("mmdp_model_set_rope: null argument");
    if (L <= 0 || L > m->cfg.max_seq_len) return set_error("mmdp_model_set_rope: L=%d exceeds max_seq_len=%d", L, m->cfg.max_seq_len);
    cudaStream_t s = (cudaStream_t)stream;
    MMDP_CUDA(cudaMemcpyAsync(m->cos_tab, cos_tab, (size_t)L * 64 * 4, cudaMemcpyDefault, s));
    MMDP_CUDA(cudaMemcpyAsync(m->sin_tab, sin_tab, (size_t)L * 64 * 4, cudaMemcpyDefault, s));
    m->rope_len = L;
    return 0;
}

MMDP_API const uint16_t* mmdp_model_hidden(mmdp_model* m) { return m ? (const uint16_t*)m->x : nullptr; }

MMDP_API int mmdp_model_error_flags(mmdp_model* m, int32_t* flags_host, void* stream) {
    if (!m || !flags_host) return set_error("mmdp_model_error_flags: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    int v = 0;
    MMDP_CUDA(cudaMemcpyAsync(&v, m->err_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    MMDP_CUDA(cudaMemsetAsync(m->err_flag, 0, sizeof(int), s));
    MMDP_CUDA(cudaStreamSynchronize(s));
    *flags_host = v;
    return 0;
}

// One of the four linears of block `l` (which: 0 = Wqkv, 1 = Wo, 2 = W13, 3 = W2) in the context's precision. FP8: the bf16
// input A is quantised into the context's e4m3 workspace (1 x 128 groups), then the e4m3 GEMM applies the same epilogue.
enum { LIN_QKV = 0, LIN_O = 1, LIN_13 = 2, LIN_2 = 3 };
static int block_linear(mmdp_model* m, const LayerWeights& l, int which, int epi, const bf16* A, int lda, int M, bf16* C, int ldc,
                        const bf16* R, int ldr, const QkvRopeArgs* qa, cudaStream_t s) {
    const int d = m->cfg.d_model, ff = m->cfg.mlp_hidden;
    const int N = which == LIN_QKV ? d + 2 * m->d_kv() : (which == LIN_13 ? 2 * ff : d);
    const int K = which == LIN_2 ? ff : d;
    if (m->precision == MMDP_PRECISION_BF16) {
        const bf16* W = which == LIN_QKV ? l.wqkv : (which == LIN_O ? l.wo : (which == LIN_13 ? l.w13 : l.w2));
        return gemm_bf16(epi, A, lda, W, K, M, N, K, C, ldc, R, ldr, qa, s);
    }
    const uint8_t* W = which == LIN_QKV ? l.wqkv8 : (which == LIN_O ? l.wo8 : (which == LIN_13 ? l.w13_8 : l.w2_8));
    const float* sw = which == LIN_QKV ? l.sqkv : (which == LIN_O ? l.so : (which == LIN_13 ? l.s13 : l.s2));
    if (quantize_fp8(A, lda, M, K, 128, m->a8, K, m->as, s)) return -1;
    return gemm_fp8(epi, m->a8, K, m->as, W, K, sw, M, N, K, C, ldc, R, ldr, qa, s);
}

// V^T pad rule. Block s of m->vt ([max_batch][Hkv][128][Lpad], the batch row or the packed sequence s) is read by the P·V MMA
// up to its padded length, and its columns [L_s, Lpad) meet P == 0 there: they must be finite zeros. A forward over blocks
// [0, n) with lengths lens[] at column stride Lpad zeroes the whole buffer when the stride changes or when one of its blocks
// holds columns beyond its new length (a longer forward wrote them); otherwise every column it reads past L_s is still zero.
static int vt_prepare(mmdp_model* m, int n, const int* lens, int Lpad, cudaStream_t s) {
    bool zero = m->vt_Lpad != Lpad;
    for (int i = 0; i < n && !zero; ++i) zero = m->vt_len[i] > lens[i];
    if (zero) {
        MMDP_CUDA(cudaMemsetAsync(m->vt, 0, (size_t)m->cfg.max_batch * m->d_kv() * m->Lpad_max * 2, s));
        m->vt_len.assign(m->cfg.max_batch, 0);
        m->vt_Lpad = Lpad;
    }
    for (int i = 0; i < n; ++i) m->vt_len[i] = lens[i];
    return 0;
}

// ln_f + LM head on the gathered rows (rows_a: all V columns; rows_b: columns [col0_b, col0_b + ncols_b)) of the M rows in
// x (m->x when null), normalised into xr (m->xr when null). row_lo / row_hi / L: the last block's row window (0: none); a row
// outside it raises bit 2 of the error flag.
static int head_rows(mmdp_model* m, int M, const int32_t* rows_a, int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b,
                     int col0_b, int ncols_b, uint16_t* out_b, int row_lo, int row_hi, int L, cudaStream_t s,
                     const bf16* x = nullptr, bf16* xr = nullptr) {
    const mmdp_model_config& c = m->cfg;
    const int d = c.d_model, V = c.vocab_size;
    if (!x) x = m->x;
    if (!xr) xr = m->xr;
    if (n_a > 0) {
        if (!rows_a || !out_a) return set_error("mmdp_model_forward: rows_a/out_a null");
        if (n_a > m->Mmax) return set_error("mmdp_model_forward: too many rows_a");
        if (rmsnorm_rows(x, d, rows_a, m->ln_f, xr, d, n_a, d, c.rms_eps, s, M, m->err_flag, row_lo, row_hi, L)) return -1;
        if (gemm_bf16(EPI_PLAIN, xr, d, m->head, d, n_a, V, d, (bf16*)out_a, V, nullptr, 0, nullptr, s)) return -1;
    }
    if (n_b > 0) {
        if (!rows_b || !out_b) return set_error("mmdp_model_forward: rows_b/out_b null");
        if (n_a + n_b > m->Mmax) return set_error("mmdp_model_forward: too many rows_a + rows_b");
        bf16* xr_b = xr + (size_t)n_a * d;
        if (rmsnorm_rows(x, d, rows_b, m->ln_f, xr_b, d, n_b, d, c.rms_eps, s, M, m->err_flag, row_lo, row_hi, L)) return -1;
        if (gemm_bf16(EPI_PLAIN, xr_b, d, m->head + (size_t)col0_b * d, d, n_b, ncols_b, d, (bf16*)out_b, ncols_b, nullptr, 0, nullptr, s)) return -1;
    }
    return 0;
}

static int model_forward(mmdp_model* m, const int64_t* ids, int B, int L, uint16_t* full_logits, const int32_t* rows_a,
                         int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b, int col0_b, int ncols_b,
                         uint16_t* out_b, int row_lo, int row_hi, void* stream) {
    if (!m || !ids) return set_error("mmdp_model_forward: null argument");
    const mmdp_model_config& c = m->cfg;
    if (B <= 0 || B > c.max_batch || L <= 0 || L > c.max_seq_len)
        return set_error("mmdp_model_forward: B=%d L=%d outside workspace (max_batch=%d max_seq_len=%d)", B, L, c.max_batch, c.max_seq_len);
    if (L > m->rope_len) return set_error("mmdp_model_forward: rotary table covers %d positions, need %d", m->rope_len, L);
    if (n_b > 0 && (col0_b < 0 || ncols_b <= 0 || col0_b + ncols_b > c.vocab_size || (ncols_b % 8)))
        return set_error("mmdp_model_forward: bad column window [%d,+%d)", col0_b, ncols_b);
    cudaStream_t s = (cudaStream_t)stream;
    const int d = c.d_model, ff = c.mlp_hidden, V = c.vocab_size, H = c.n_heads, Hkv = m->n_kv_heads, dkv = m->d_kv();
    const int M = B * L;
    const int Lpad = ((L + 7) / 8) * 8;
    const std::vector<int> lens(B, L);
    if (vt_prepare(m, B, lens.data(), Lpad, s)) return -1;
    const float scale = 1.0f / sqrtf(128.0f);
    if (embed_rows(ids, m->wte, m->x, M, d, V, s, m->err_flag)) return -1;
    QkvRopeArgs qa{m->q, m->k, m->vt, m->cos_tab, m->sin_tab, L, Lpad, d, H};
    qa.n_kv_heads = Hkv;
    const int qkv_epi = m->gqa() ? EPI_QKVGQA : EPI_QKVROPE;
    // Row window of the LAST block: nothing after the last block mixes rows (ln_f and the LM head are row-wise and only the rows in
    // rows_a / rows_b are read), so its query rows / attn_out / MLP outside positions [row_lo, row_hi) of every batch row are dead
    // work: the keys and values of ALL rows are still computed, the rest of the block runs on the window only (per batch row).
    const bool window = !full_logits && opt(OPT_ROW_WINDOW) && row_hi > row_lo && row_lo >= 0 && row_hi <= L && (row_hi - row_lo) < L;  // MMDP_ROW_WINDOW=0: A/B switch
    if (!window) { row_lo = 0; row_hi = L; }
    for (int li = 0; li < c.n_layers; ++li) {
        const LayerWeights& l = m->layers[li];
        const bool win = window && li == c.n_layers - 1;
        qa.bias = l.qkv_bias;
        if (rmsnorm(m->x, d, l.attn_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (block_linear(m, l, LIN_QKV, qkv_epi, m->xn, d, M, nullptr, 0, nullptr, 0, &qa, s)) return -1;
        if (!win) {
            if (attention_fwd(m->q, m->k, m->vt, m->att, B, H, L, Lpad, scale, s, 0, Hkv)) return -1;
            if (block_linear(m, l, LIN_O, EPI_RESID, m->att, d, M, m->x, d, m->x, d, nullptr, s)) return -1;
            if (rmsnorm(m->x, d, l.ff_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
            if (block_linear(m, l, LIN_13, EPI_SWIGLU, m->xn, d, M, m->h, ff, nullptr, 0, nullptr, s)) return -1;
            if (block_linear(m, l, LIN_2, EPI_RESID, m->h, ff, M, m->x, d, m->x, d, nullptr, s)) return -1;
            continue;
        }
        const int Mw = row_hi - row_lo;
        for (int b = 0; b < B; ++b) {  // one row range per batch row (B = 1, or the CFG batch of variant M)
            const size_t r0 = (size_t)b * L + row_lo, o_d = r0 * d, o_ff = r0 * ff;
            if (attention_fwd(m->q + o_d, m->k + (size_t)b * L * dkv, m->vt + (size_t)b * Hkv * 128 * Lpad, m->att + o_d, 1, H, L, Lpad, scale, s, Mw,
                              Hkv)) return -1;
            if (block_linear(m, l, LIN_O, EPI_RESID, m->att + o_d, d, Mw, m->x + o_d, d, m->x + o_d, d, nullptr, s)) return -1;
            if (rmsnorm(m->x + o_d, d, l.ff_norm, m->xn + o_d, d, Mw, d, c.rms_eps, s)) return -1;
            if (block_linear(m, l, LIN_13, EPI_SWIGLU, m->xn + o_d, d, Mw, m->h + o_ff, ff, nullptr, 0, nullptr, s)) return -1;
            if (block_linear(m, l, LIN_2, EPI_RESID, m->h + o_ff, ff, Mw, m->x + o_d, d, m->x + o_d, d, nullptr, s)) return -1;
        }
    }
    if (full_logits) {
        if (rmsnorm(m->x, d, m->ln_f, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_PLAIN, m->xn, d, m->head, d, M, V, d, (bf16*)full_logits, V, nullptr, 0, nullptr, s)) return -1;
    }
    return head_rows(m, M, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, window ? row_lo : 0, window ? row_hi : 0,
                     window ? L : 0, s);
}

// Token-cache forward (reference: LLaDAModelLM.forward(input_ids, use_cache=True, to_compute_mask=mask, cat=key),
// MMaDA-Parallel-A/model/modeling_llada.py:1244-1245 (ids restricted to the masked positions), :929-940 (per-block k / v caches,
// scattered at the recomputed positions), :715-716 + :412-435 (rotary with the recomputed tokens' own positions for q, all
// positions for k), :1406-1413 (logit cache). One call computes the Tq selected tokens of every batch row against the FULL
// cached key/value set:
//   ids       [B * Tq]      the selected tokens' ids, batch row major (pos_map == NULL: Tq == L, every token - a full forward)
//   pos_map   [B * Tq]      their positions inside the sequence (int32; increasing per batch row), or NULL
//   kcache    [n_layers][B * L][d]            keys AFTER rotary (rope(k, pos) is a function of the cached value and its
//                                              position only, so caching it is equivalent to the reference's rope of the cached k)
//   vtcache   [n_layers][B][H][128][Lpad]     values, transposed; pad columns must be zero (Lpad = L rounded up to 8)
//   logits    [B * Tq][V]   logits of the selected tokens (the caller scatters them into its logit cache)
// The selected tokens' k / v^T are written into the caches at their positions before attention, like the reference does.
MMDP_API int mmdp_model_forward(mmdp_model* m, const int64_t* ids, int B, int L, uint16_t* full_logits, const int32_t* rows_a,
                       int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b, int col0_b, int ncols_b,
                       uint16_t* out_b, void* stream) {
    return model_forward(m, ids, B, L, full_logits, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, 0, 0, stream);
}
MMDP_API int mmdp_model_forward_window(mmdp_model* m, const int64_t* ids, int B, int L, const int32_t* rows_a, int n_a, uint16_t* out_a,
                              const int32_t* rows_b, int n_b, int col0_b, int ncols_b, uint16_t* out_b, int row_lo, int row_hi,
                              void* stream) {
    return model_forward(m, ids, B, L, nullptr, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, row_lo, row_hi, stream);
}

// Packed forward; win_lo / win_hi (host, both null or both set): the last block's row window [win_lo[s], win_hi[s]) of every
// sequence s. Layers 0 .. n-2 and the last block's norm + QKV run on all M packed rows (keys and values of every row). With
// windows, the window rows of x are then gathered into m->xr, and the rest of the last block (attention, attn_out + residual,
// ff_norm, SwiGLU, ff_out + residual) runs on those Mw compact rows; the head reads them through the row map (ln_f into m->xn).
// m->x then keeps the input of the last block.
static int forward_packed(mmdp_model* m, const int64_t* ids, int n_seg, const int32_t* seg_len, const int32_t* win_lo,
                          const int32_t* win_hi, const int32_t* rows_a, int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b,
                          int col0_b, int ncols_b, uint16_t* out_b, void* stream) {
    if (!m || !ids || !seg_len) return set_error("mmdp_model_forward_packed: null argument");
    const mmdp_model_config& c = m->cfg;
    if (n_seg <= 0 || n_seg > c.max_batch || n_seg > kMaxSegs)
        return set_error("mmdp_model_forward_packed: %d sequences outside [1, %d] (max_batch, at most %d)", n_seg, c.max_batch, kMaxSegs);
    if (!win_lo != !win_hi) return set_error("mmdp_model_forward_packed_window: give both win_lo and win_hi, or neither");
    SegTable segs{};
    segs.n = n_seg;
    int Lmax = 0;
    for (int i = 0; i < n_seg; ++i) {
        if (seg_len[i] <= 0 || seg_len[i] > c.max_seq_len)
            return set_error("mmdp_model_forward_packed: sequence %d has length %d (max_seq_len=%d)", i, seg_len[i], c.max_seq_len);
        if (win_lo && (win_lo[i] < 0 || win_lo[i] >= win_hi[i] || win_hi[i] > seg_len[i]))
            return set_error("mmdp_model_forward_packed_window: sequence %d of length %d has the window [%d, %d)", i, seg_len[i],
                             win_lo[i], win_hi[i]);
        segs.start[i + 1] = segs.start[i] + seg_len[i];
        Lmax = seg_len[i] > Lmax ? seg_len[i] : Lmax;
    }
    if (Lmax > m->rope_len) return set_error("mmdp_model_forward_packed: rotary table covers %d positions, need %d", m->rope_len, Lmax);
    if (n_b > 0 && (col0_b < 0 || ncols_b <= 0 || col0_b + ncols_b > c.vocab_size || (ncols_b % 8)))
        return set_error("mmdp_model_forward_packed: bad column window [%d,+%d)", col0_b, ncols_b);
    // windows that cover whole sequences skip nothing; MMDP_ROW_WINDOW=0 switches them off (A/B switch)
    WinTable wt{};
    bool window = false;
    if (win_lo && opt(OPT_ROW_WINDOW)) {
        wt.n = n_seg;
        for (int i = 0; i < n_seg; ++i) {
            wt.start[i + 1] = segs.start[i + 1];
            wt.lo[i] = win_lo[i];
            wt.hi[i] = win_hi[i];
            wt.out0[i + 1] = wt.out0[i] + win_hi[i] - win_lo[i];
            window = window || win_hi[i] - win_lo[i] < seg_len[i];
        }
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int d = c.d_model, ff = c.mlp_hidden, V = c.vocab_size, H = c.n_heads, Hkv = m->n_kv_heads;
    const int M = segs.start[n_seg], Mw = window ? wt.out0[n_seg] : M;
    const int Lpad = ((Lmax + 7) / 8) * 8;
    if (vt_prepare(m, n_seg, seg_len, Lpad, s)) return -1;
    if (packed_row_map(segs, m->seg_pos, s)) return -1;
    const float scale = 1.0f / sqrtf(128.0f);
    if (embed_rows(ids, m->wte, m->x, M, d, V, s, m->err_flag)) return -1;
    QkvRopeArgs qa{m->q, m->k, m->vt, m->cos_tab, m->sin_tab, Lmax, Lpad, d, H};
    qa.seg_pos = m->seg_pos;
    qa.n_kv_heads = Hkv;
    const int qkv_epi = m->gqa() ? EPI_QKVGQA_PACKED : EPI_QKVROPE_PACKED;
    for (int li = 0; li < c.n_layers; ++li) {
        const LayerWeights& l = m->layers[li];
        const bool win = window && li == c.n_layers - 1;
        bf16* x = win ? m->xr : m->x;  // the residual stream of the rows this block finishes, Mb of them
        const int Mb = win ? Mw : M;
        qa.bias = l.qkv_bias;
        if (rmsnorm(m->x, d, l.attn_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (block_linear(m, l, LIN_QKV, qkv_epi, m->xn, d, M, nullptr, 0, nullptr, 0, &qa, s)) return -1;
        if (win) {
            if (window_gather(wt, m->x, m->xr, d, s)) return -1;
            if (attention_packed_fwd(m->q, m->k, m->vt, m->att, segs, H, Lpad, scale, s, Hkv, wt.lo, wt.hi)) return -1;
        } else {
            if (attention_packed_fwd(m->q, m->k, m->vt, m->att, segs, H, Lpad, scale, s, Hkv)) return -1;
        }
        if (block_linear(m, l, LIN_O, EPI_RESID, m->att, d, Mb, x, d, x, d, nullptr, s)) return -1;
        if (rmsnorm(x, d, l.ff_norm, m->xn, d, Mb, d, c.rms_eps, s)) return -1;
        if (block_linear(m, l, LIN_13, EPI_SWIGLU, m->xn, d, Mb, m->h, ff, nullptr, 0, nullptr, s)) return -1;
        if (block_linear(m, l, LIN_2, EPI_RESID, m->h, ff, Mb, x, d, x, d, nullptr, s)) return -1;
    }
    if (!window) return head_rows(m, M, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, 0, 0, 0, s);
    if (n_a + n_b > m->Mmax) return set_error("mmdp_model_forward_packed_window: too many rows_a + rows_b");
    if ((n_a > 0 && !rows_a) || (n_b > 0 && !rows_b)) return set_error("mmdp_model_forward_packed_window: rows_a/rows_b null");
    if (window_row_map(wt, rows_a, n_a, m->win_rows, m->err_flag, s)) return -1;
    if (window_row_map(wt, rows_b, n_b, m->win_rows + n_a, m->err_flag, s)) return -1;
    return head_rows(m, Mw, m->win_rows, n_a, out_a, m->win_rows + n_a, n_b, col0_b, ncols_b, out_b, 0, 0, 0, s, m->xr, m->xn);
}

MMDP_API int mmdp_model_forward_packed(mmdp_model* m, const int64_t* ids, int n_seg, const int32_t* seg_len, const int32_t* rows_a,
                                       int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b, int col0_b, int ncols_b, uint16_t* out_b,
                                       void* stream) {
    return forward_packed(m, ids, n_seg, seg_len, nullptr, nullptr, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, stream);
}

MMDP_API int mmdp_model_forward_packed_window(mmdp_model* m, const int64_t* ids, int n_seg, const int32_t* seg_len, const int32_t* win_lo,
                                              const int32_t* win_hi, const int32_t* rows_a, int n_a, uint16_t* out_a, const int32_t* rows_b,
                                              int n_b, int col0_b, int ncols_b, uint16_t* out_b, void* stream) {
    return forward_packed(m, ids, n_seg, seg_len, win_lo, win_hi, rows_a, n_a, out_a, rows_b, n_b, col0_b, ncols_b, out_b, stream);
}

MMDP_API int mmdp_model_forward_cached(mmdp_model* m, const int64_t* ids, int B, int L, int Tq, const int32_t* pos_map, uint16_t* kcache,
                              uint16_t* vtcache, uint16_t* logits, void* stream) {
    if (!m || !ids || !kcache || !vtcache) return set_error("mmdp_model_forward_cached: null argument");
    const mmdp_model_config& c = m->cfg;
    if (B <= 0 || B > c.max_batch || L <= 0 || L > c.max_seq_len || Tq <= 0 || Tq > L)
        return set_error("mmdp_model_forward_cached: B=%d L=%d Tq=%d outside workspace (max_batch=%d max_seq_len=%d)", B, L, Tq, c.max_batch, c.max_seq_len);
    if (!pos_map && Tq != L) return set_error("mmdp_model_forward_cached: a partial forward needs the position map");
    if (m->gqa()) return set_error("mmdp_model_forward_cached: the token cache holds d_model-wide multi-head keys without a q/k/v bias");
    if (L > m->rope_len) return set_error("mmdp_model_forward_cached: rotary table covers %d positions, need %d", m->rope_len, L);
    cudaStream_t s = (cudaStream_t)stream;
    const int d = c.d_model, ff = c.mlp_hidden, V = c.vocab_size, H = c.n_heads;
    const int M = B * Tq;
    const int Lpad = ((L + 7) / 8) * 8;
    const float scale = 1.0f / sqrtf(128.0f);
    const size_t k_layer = (size_t)B * L * d, vt_layer = (size_t)B * d * Lpad;
    if (embed_rows(ids, m->wte, m->x, M, d, V, s, m->err_flag)) return -1;
    for (int li = 0; li < c.n_layers; ++li) {
        const LayerWeights& l = m->layers[li];
        bf16* kc = (bf16*)kcache + (size_t)li * k_layer;
        bf16* vc = (bf16*)vtcache + (size_t)li * vt_layer;
        QkvRopeArgs qa{m->q, kc, vc, m->cos_tab, m->sin_tab, L, Lpad, d, H, pos_map, pos_map ? Tq : 0};
        if (rmsnorm(m->x, d, l.attn_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (block_linear(m, l, LIN_QKV, EPI_QKVROPE, m->xn, d, M, nullptr, 0, nullptr, 0, &qa, s)) return -1;
        if (attention_fwd(m->q, kc, vc, m->att, B, H, L, Lpad, scale, s, Tq)) return -1;
        if (block_linear(m, l, LIN_O, EPI_RESID, m->att, d, M, m->x, d, m->x, d, nullptr, s)) return -1;
        if (rmsnorm(m->x, d, l.ff_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (block_linear(m, l, LIN_13, EPI_SWIGLU, m->xn, d, M, m->h, ff, nullptr, 0, nullptr, s)) return -1;
        if (block_linear(m, l, LIN_2, EPI_RESID, m->h, ff, M, m->x, d, m->x, d, nullptr, s)) return -1;
    }
    if (logits) {
        if (rmsnorm(m->x, d, m->ln_f, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_PLAIN, m->xn, d, m->head, d, M, V, d, (bf16*)logits, V, nullptr, 0, nullptr, s)) return -1;
    }
    return 0;
}

}  // extern "C"
