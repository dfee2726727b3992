// Internal (C++) declarations shared by the .cu translation units behind the C ABI in include/mmdp.h.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace mmdp {

// EPI_QKVROPE_PACKED: EPI_QKVROPE over a packed variable-length batch (QkvRopeArgs::seg_pos)
// EPI_QKVGQA / EPI_QKVGQA_PACKED: the same two with grouped-query k / v (n_kv_heads <= n_heads) and an optional q / k / v bias;
// the multi-head instantiations above stay free of both
enum Epilogue { EPI_PLAIN = 0, EPI_RESID = 1, EPI_QKVROPE = 2, EPI_SWIGLU = 3, EPI_F32 = 4, EPI_QKVROPE_PACKED = 5,
                EPI_QKVGQA = 6, EPI_QKVGQA_PACKED = 7 };
constexpr bool epi_is_gqa(int epi) { return epi == EPI_QKVGQA || epi == EPI_QKVGQA_PACKED; }
constexpr bool epi_is_qkv(int epi) { return epi == EPI_QKVROPE || epi == EPI_QKVROPE_PACKED || epi_is_gqa(epi); }
constexpr bool epi_is_packed(int epi) { return epi == EPI_QKVROPE_PACKED || epi == EPI_QKVGQA_PACKED; }

// Packed variable-length batch: sequence s occupies rows [start[s], start[s + 1]) of one packed row space; attention never
// crosses from one sequence into another and positions restart at 0 in each. kMaxSegs bounds the sequences of one launch
// (the table travels as a kernel parameter).
static constexpr int kMaxSegs = 64;
struct SegTable {
    int n;
    int start[kMaxSegs + 1];
};

int set_error(const char* fmt, ...);  // records the message for mmdp_last_error(), returns -1
const char* last_error();
int num_sms();

// Per-launch accounting. Every kernel launch of this library goes through a LaunchScope: it bumps the launch counter
// and, when profiling is enabled (bench.py's roofline pass), brackets the launch with CUDA events on the launching stream.
enum LaunchKind { LK_GEMM = 0, LK_ATTN = 1, LK_ROW = 2, LK_SAMPLE = 3, LK_COUNT = 4 };
struct LaunchScope {
    LaunchScope(int kind, double work, cudaStream_t s);
    ~LaunchScope();
    int idx;
    cudaStream_t stream;
};
void prof_enable(int on);
int prof_summary(double* ms, double* work, long long* launches);  // arrays of LK_COUNT; synchronises the device
long long launch_count(int reset);

// Launch options of the library (runtime.cu). pdl: consecutive kernels of a forward are launched with programmatic
// stream serialization (MMDP_PDL=0 disables); every kernel launched through launch_ex with pdl=true calls pdl_wait().
int pdl_mode();
void set_pdl_mode(int on);
int env_int(const char* name, int dflt);
// tuning options (runtime.cu): environment default, mmdp_set_option(key, value) at run time
enum OptId { OPT_PDL = 0, OPT_GEMM_SPLITK, OPT_GEMM_L2PF, OPT_GEMM_L2PF_MOD, OPT_GEMM_GROUP_M, OPT_ATTN_SPLIT_TAIL,
             OPT_RMSNORM_WARP, OPT_ROW_WINDOW, OPT_ATTN_VERSION, OPT_GEMM_PAIR, OPT_COUNT };
int opt(int id);
int set_opt(const char* key, int value);

// cudaLaunchKernelEx wrapper: optional programmatic dependent launch and/or cooperative (co-residency guaranteed) launch.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                             bool coop, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[2];
    unsigned n = 0;
    if (pdl) {
        at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (coop) {
        at[n].id = cudaLaunchAttributeCooperative;
        at[n].val.cooperative = 1;
        ++n;
    }
    cfg.attrs = at;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#define MMDP_CUDA(expr)                                                                              \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess)                                                                       \
            return ::mmdp::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)

// 2-D bf16 tensor map: tensor [rows, cols] with row stride ld (elements), box [box_rows, box_cols],
// 128-byte swizzle (box_cols must be 64), out-of-bounds elements read as zero.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                      uint32_t box_cols);
// generic: elem_bytes 1 (e4m3, box_cols 128), 2 (bf16, box_cols 64) or 4 (fp32/tf32, box_cols 32)
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols);

// TF32 shifted-tap GEMM (conv engine) and the decoder's row kernels (conv_tf32.cu)
int conv_tf32(const float* A, int lda, long long a_rows, const float* W, int M, int N, int K, int T, const int* shifts,
              float* C, int ldc, const float* R, int ldr, const float* bias, int bias_along_m, float alpha, int pad_w,
              int pad_h, int scatter_w, int scatter_h, cudaStream_t stream);
int gn_swish(const float* x, float* y, int B, int C, int H, int W, double* stats_ws, const float* gamma, const float* beta,
             float eps, int swish, int compact, cudaStream_t stream);
int upsample2x(const float* x, float* y, int B, int C, int H, int W, cudaStream_t stream);
int softmax_rows_ld(float* s, int rows, int n, int ld, cudaStream_t stream);
int zero_border(float* y, int B, int C, int H, int W, cudaStream_t stream);
int lfq_to_padded(const int64_t* ids, float* z, int B, int H, int W, int bits, int Cpad, cudaStream_t stream);
int nchw_to_padded(const float* x, float* y, int B, int C, int Cpad, int H, int W, cudaStream_t stream);
int downsample_pick(const float* src, float* dst, int B, int C, int H, int W, cudaStream_t stream);
int lfq_indices(const float* z, int64_t* ids, int B, int h, int w, int bits, int ld, cudaStream_t stream);
int padded_to_nchw(const float* x, float* y, int B, int C, int ld, int H, int W, cudaStream_t stream);
// learned codebook of the aMUSEd VQ-VAE (vq_codebook.cu). codebook_to_padded: ids outside [0, n_codes) raise bit 0 of *err
// and give zero vectors. vq_nearest: argmin_k |z - e_k|^2 in exact fp32, lowest index on ties; zq (nullable) NCHW.
int codebook_to_padded(const int64_t* ids, const float* cb, float* z, int B, int h, int w, int C, int Cpad, int64_t n_codes,
                       int* err, cudaStream_t stream);
int vq_nearest(const float* z, const float* cb, int B, int C, int h, int w, int n_codes, int64_t* ids, float* zq,
               cudaStream_t stream);

struct QkvRopeArgs {
    __nv_bfloat16* q;       // [B*L, d_model]   rotary applied, head h at columns [128h, 128h+128)
    __nv_bfloat16* k;       // [B*L, d_model]   rotary applied
    __nv_bfloat16* vt;      // [B, H, 128, Lpad] V transposed (token index contiguous); pad columns must stay zero
    const float* cos_tab;   // [L, 64] fp32
    const float* sin_tab;   // [L, 64] fp32
    int L, Lpad, d_model, n_heads;
    const int* pos_map = nullptr;  // token-cache forward: compact row r = token pos_map[r] of batch row r / Tq (k, v^T scattered to it)
    int Tq = 0;
    int chunked = 0;  // 1: the launch covers a row range of the [B*L] sequence (M need not be a multiple of L)
    int row0 = 0;  // GEMM row r is token row0 + r of the flattened [B*L] sequence (row-chunked tensor-parallel forward); q / k point at that row
    const int2* seg_pos = nullptr;  // EPI_QKVROPE_PACKED: row r is token seg_pos[r].y of sequence seg_pos[r].x (q / k stay at row r,
                                    // v^T goes to vt[seg][head][d][pos]); L is then the longest sequence
    // EPI_QKVGQA*: GEMM columns [0, d) = q, [d, d + d_kv) = k, [d + d_kv, d + 2 d_kv) = v with d_kv = 128 n_kv_heads; k is
    // [rows, d_kv], vt [B, n_kv_heads, 128, Lpad]. bias (nullable): bf16 [d + 2 d_kv], added before the first bf16 rounding
    int n_kv_heads = 0;
    const __nv_bfloat16* bias = nullptr;
};

// device map of a packed batch: seg_pos[r] = (sequence, position) of packed row r, for the rows of `segs`
int packed_row_map(const SegTable& segs, int2* seg_pos, cudaStream_t stream);

// EPI_F32 only: push the fp32 partial rows to their owners' receive buffers instead of storing them to C (tensor parallel)
struct GemmScatter {
    float* dst[8];  // peer-mapped receive buffer of every rank: [n_ranks][rows_per_rank][ldc] fp32
    int rows_per_rank, slot;
};

int gemm_bf16(int epi, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, int M, int N, int K,
              __nv_bfloat16* C, int ldc, const __nv_bfloat16* resid, int ldr, const QkvRopeArgs* qa,
              cudaStream_t stream, const GemmScatter* sc = nullptr);

// tile order of the persistent GEMMs (gemm.cu): the m-tile group size for M rows
int gemm_group_m(int M);

// FP8 (e4m3) path (fp8.cu). quantize_fp8: x bf16 [rows, K] (row stride ldx) -> q e4m3 [rows, K] (row stride ldq) and fp32
// scales [K / group][rows]; group divides K and is a multiple of 128. gemm_fp8: A e4m3 [M, K] with scales sa [K/128][M],
// W e4m3 [N, K] with row scales sw [N]; epilogues PLAIN, RESID, SWIGLU (W13 interleaved in 64-row blocks), QKVROPE / QKVGQA,
// and F32 (fp32 C, or with `scat` each row pushed to the rank that owns it, as gemm_bf16's scatter).
int quantize_fp8(const __nv_bfloat16* x, int ldx, int rows, int K, int group, uint8_t* q, int ldq, float* scales,
                 cudaStream_t stream);
int gemm_fp8(int epi, const uint8_t* A, int lda, const float* sa, const uint8_t* W, int ldw, const float* sw, int M, int N,
             int K, __nv_bfloat16* C, int ldc, const __nv_bfloat16* resid, int ldr, const QkvRopeArgs* qa, cudaStream_t stream,
             const GemmScatter* scat = nullptr);

int gemm_pair_mode();
void set_gemm_pair_mode(int on);
int gemm_splitk_mode();
void set_gemm_splitk_mode(int mode);

// Lq > 0: q / out hold Lq query rows per batch row (a compact subset), k / vt the full L keys (token-cache forward).
// Hkv > 0 (grouped-query attention, H % Hkv == 0): k [B * L, 128 Hkv], vt [B, Hkv, 128, Lpad]; query head h reads kv head
// h / (H / Hkv). 0 = H.
int attention_fwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out, int B,
                  int H, int L, int Lpad, float scale, cudaStream_t stream, int Lq = 0, int Hkv = 0);
// packed variable-length batch: q / out [segs.start[n], H * 128], k [segs.start[n], Hkv * 128], vt [segs.n, Hkv, 128, Lpad];
// columns [L_s, Lpad) of sequence s's V^T block must be finite zeros.
// win_lo / win_hi (host arrays, both or neither): sequence s computes its query rows [win_lo[s], win_hi[s]) only, against all of
// its keys, and out holds the windows end to end (sum of hi - lo rows); 0 <= lo < hi <= L_s
int attention_packed_fwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out,
                         const SegTable& segs, int H, int Lpad, float scale, cudaStream_t stream, int Hkv = 0,
                         const int* win_lo = nullptr, const int* win_hi = nullptr);

// err (nullable): device int, bit 0 is raised when an id is outside [0, vocab) (the kernel then reads row 0)
int embed_rows(const int64_t* ids, const __nv_bfloat16* wte, __nv_bfloat16* x, int M, int d, int64_t vocab,
               cudaStream_t stream, int* err = nullptr);
int rmsnorm(const __nv_bfloat16* x, int ldx, const __nv_bfloat16* w, __nv_bfloat16* y, int ldy, int M, int d, float eps,
            cudaStream_t stream);
int resid_add_f32(__nv_bfloat16* x, int ldx, const float* partial, int ldp, int M, int d, cudaStream_t stream);
// src_rows / err: gather indices outside [0, src_rows) raise bit 1 of *err (nullable) and read row 0
int rmsnorm_rows(const __nv_bfloat16* x, int ldx, const int* rows, const __nv_bfloat16* w, __nv_bfloat16* y, int ldy,
                 int M, int d, float eps, cudaStream_t stream, int src_rows = 0x7fffffff, int* err = nullptr, int row_lo = 0, int row_hi = 0, int row_mod = 0);

int text_step(const __nv_bfloat16* cond, const __nv_bfloat16* uncond, int64_t ld, int R, int V, float text_cfg,
              const __nv_bfloat16* unoise, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
              int k, int64_t* x0_ws, double* conf_ws, cudaStream_t stream, const double* unoise64 = nullptr);
int image_step(int variant, const __nv_bfloat16* cond, const __nv_bfloat16* unc_a, const __nv_bfloat16* unc_b, int64_t ld,
               int N, int C, float s_a, float s_b, const __nv_bfloat16* qnoise, const __nv_bfloat16* conf_noise,
               float temp, int sched_len, int64_t* ids, const int* pos, int64_t mask_id, int64_t vq_offset,
               int32_t* sampled_ws, float* selp_ws, uint8_t* unknown_ws, __nv_bfloat16* probs_out,
               int32_t* mask_len_out, uint8_t* masking_out, cudaStream_t stream);
int image_remask(int variant, int N, const int32_t* sampled, const float* selp, const uint8_t* unknown,
                 const __nv_bfloat16* conf_noise, float temp, int sched_len, int64_t* ids, const int* pos, int64_t mask_id,
                 int64_t vq_offset, int32_t* mask_len_out, uint8_t* masking_out, cudaStream_t stream, int k_direct = -1);
int image_step_t2i(const __nv_bfloat16* cond, const __nv_bfloat16* uncond, int64_t ld, int N, int C, float cfg,
                   const __nv_bfloat16* gumbel_u, float tau, const __nv_bfloat16* conf_u, float temperature, int keep_n,
                   int64_t* ids, const int* pos, int64_t mask_id, int64_t vq_offset, int32_t* sampled_ws, float* selp_ws,
                   uint8_t* unknown_ws, uint8_t* masking_out, cudaStream_t stream);
int lfq_decode(const int64_t* ids, float* zq, int B, int N, int bits, cudaStream_t stream);
// tensor-parallel collective over NVLink peer memory (tp_collective.cu)
int tp_reduce_norm(const float* recv_local, int rows_per_rank, int n_src, uint16_t* const* xn, uint32_t* const* flags, int n_ranks,
                   int my_rank, uint16_t* x_shard, const uint16_t* w, int row0, int nrows, int d, float eps, uint32_t epoch,
                   unsigned int* done_counter, cudaStream_t stream);
// FP8 form: the normalised rows go to every rank as e4m3 bytes xq[r] [rows, d] plus 1 x 128 group scales xs[r] [d / 128][ld_s],
// bitwise what quantize_fp8(group 128) makes of the bf16 rows tp_reduce_norm would store
int tp_reduce_norm_fp8(const float* recv_local, int rows_per_rank, int n_src, uint8_t* const* xq, float* const* xs, int ld_s,
                       uint32_t* const* flags, int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* w, int row0, int nrows,
                       int d, float eps, uint32_t epoch, unsigned int* done_counter, cudaStream_t stream);

}  // namespace mmdp
