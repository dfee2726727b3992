// extern "C" surface (include/mmdp.h) and the native model context: device-resident packed weights, activation
// workspace and the per-layer launch sequence of LLaDAModel.forward (MMaDA-Parallel-A/model/modeling_llada.py:1201-1415,
// block :906-972). No torch types cross this boundary.
#include "../../include/mmdp.h"
#include "mmdp_internal.h"

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
    bf16* wqkv;       // [3d, d]   rows: q_proj | k_proj | v_proj
    bf16* wo;         // [d, d]
    bf16* w13;        // [2ff, d]  128-row blocks interleaved: ff_proj block t, up_proj block t
    bf16* w2;         // [d, ff]
    bf16* attn_norm;  // [d]
    bf16* ff_norm;    // [d]
};

struct mmdp_model {
    mmdp_model_config cfg;
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
    int* err_flag = nullptr;  // device: bit 0 = token id out of range, bit 1 = logits row index out of range
    int vt_B = 0, vt_Lpad = 0, vt_L = 0;  // layout / length the vt buffer was last zeroed for
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

MMDP_API int mmdp_qkv_rope(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads, int L, int Lpad,
                  const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_model, n_heads};
    return gemm_bf16(EPI_QKVROPE, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, 3 * d_model, d_model, nullptr, 0,
                     nullptr, 0, &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_qkv_rope_tp(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads_local, int L,
                      int Lpad, const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream) {
    const int d_attn = n_heads_local * 128;
    QkvRopeArgs qa{(bf16*)q, (bf16*)k, (bf16*)vt, cos_tab, sin_tab, L, Lpad, d_attn, n_heads_local};
    return gemm_bf16(EPI_QKVROPE, (const bf16*)A, lda, (const bf16*)Wqkv, d_model, M, 3 * d_attn, d_model, nullptr, 0, nullptr, 0,
                     &qa, (cudaStream_t)stream);
}

MMDP_API int mmdp_resid_add_f32(uint16_t* x, int ldx, const float* partial, int ldp, int M, int d, void* stream) {
    return resid_add_f32((bf16*)x, ldx, partial, ldp, M, d, (cudaStream_t)stream);
}

MMDP_API int mmdp_attention(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, int n_heads, int L,
                   int Lpad, float scale, void* stream) {
    return attention_fwd((const bf16*)q, (const bf16*)k, (const bf16*)vt, (bf16*)out, B, n_heads, L, Lpad, scale,
                         (cudaStream_t)stream);
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
    if (rows_per_rank <= 0 || (M + rows_per_rank - 1) / rows_per_rank > n_ranks) return set_error("mmdp_gemm_f32_scatter: M does not fit n_ranks x rows_per_rank");
    GemmScatter sc{};
    for (int r = 0; r < n_ranks; ++r) sc.dst[r] = recv[r];
    sc.rows_per_rank = rows_per_rank; sc.slot = slot;
    return gemm_bf16(EPI_F32, (const bf16*)A, lda, (const bf16*)W, ldw, M, N, K, nullptr, N, nullptr, 0, nullptr, (cudaStream_t)stream, &sc);
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

MMDP_API int mmdp_tp_forward(const mmdp_tp_ctx* c, const int64_t* ids, int B, int L, uint32_t epoch0, uint32_t* epoch_out, void* stream) {
    if (!c || !ids || !epoch_out) return set_error("mmdp_tp_forward: null argument");
    cudaStream_t s0 = (cudaStream_t)stream;
    const int d = c->d_model, Hl = c->n_heads_local, da = Hl * 128, ffl = c->ff_local, tp = c->n_ranks;
    const int M = B * L, Lpad = ((L + 7) / 8) * 8;
    const int nch = c->n_chunks == 2 ? 2 : 1;
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
    for (int ci = 0; ci < nch; ++ci)
        for (int r = 0; r < tp; ++r) xn_chunk[ci][r] = c->xn[r] + (size_t)ch[ci].m0 * d;
    auto reduce = [&](int ci, int buf, const uint16_t* w, uint32_t ep) -> int {
        const Chunk& k = ch[ci];
        const mmdp_tp_chunk& cc = c->chunk[ci];
        return tp_reduce_norm(buf >= 0 ? cc.recv[buf][c->rank] : nullptr, k.R, buf >= 0 ? tp : 0, xn_chunk[ci], cc.flags, tp, c->rank, cc.x_shard, w,
                              k.row0, k.nrows, d, c->rms_eps, ep, cc.done_counter, k.s);
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
    if (fork()) return -1;
    ++epoch;
    for (int ci = 0; ci < nch; ++ci) {
        const Chunk& k = ch[ci];
        if (embed_rows(ids + k.m0 + k.row0, (const bf16*)c->wte, (bf16*)c->chunk[ci].x_shard, k.nrows, d, c->vocab, k.s, nullptr)) return -1;
        if (reduce(ci, -1, c->layers[0].attn_norm, epoch)) return -1;
    }
    for (int li = 0; li < c->n_layers; ++li) {
        const mmdp_tp_layer& l = c->layers[li];
        for (int ci = 0; ci < nch; ++ci) {
            const Chunk& k = ch[ci];
            QkvRopeArgs qa{(bf16*)c->q + (size_t)k.m0 * da, (bf16*)c->k + (size_t)k.m0 * da, (bf16*)c->vt, c->cos_tab, c->sin_tab, L, Lpad, da, Hl};
            qa.chunked = nch > 1; qa.row0 = k.m0;
            if (gemm_bf16(EPI_QKVROPE, xn + (size_t)k.m0 * d, d, (const bf16*)l.wqkv, d, k.Mc, 3 * da, d, nullptr, 0, nullptr, 0, &qa, k.s)) return -1;
        }
        // attention mixes all rows: both chunks' q / k / v^T must be complete, and it must be complete before either chain goes on
        if (join()) return -1;
        if (attention_fwd((const bf16*)c->q, (const bf16*)c->k, (const bf16*)c->vt, (bf16*)c->att, B, Hl, L, Lpad, scale, s0)) return -1;
        if (fork()) return -1;
        const uint32_t e1 = ++epoch, e2 = ++epoch;
        for (int ci = 0; ci < nch; ++ci) {
            const Chunk& k = ch[ci];
            const bf16* att = (const bf16*)c->att + (size_t)k.m0 * da;
            bf16* h = (bf16*)c->h + (size_t)k.m0 * ffl;
            if (gemm_bf16(EPI_F32, att, da, (const bf16*)l.wo, da, k.Mc, d, da, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[0])) return -1;
            if (reduce(ci, 0, l.ff_norm, e1)) return -1;
            if (gemm_bf16(EPI_SWIGLU, xn + (size_t)k.m0 * d, d, (const bf16*)l.w13, d, k.Mc, 2 * ffl, d, h, ffl, nullptr, 0, nullptr, k.s)) return -1;
            if (gemm_bf16(EPI_F32, h, ffl, (const bf16*)l.w2, ffl, k.Mc, d, ffl, nullptr, d, nullptr, 0, nullptr, k.s, &k.sc[1])) return -1;
            if (reduce(ci, 1, li + 1 < c->n_layers ? c->layers[li + 1].attn_norm : c->ln_f, e2)) return -1;
        }
    }
    if (join()) return -1;
    *epoch_out = epoch;
    return 0;
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
    if (!c || !out) return set_error("mmdp_model_create: null argument");
    if (c->d_model != c->n_heads * 128) return set_error("mmdp_model_create: head_dim must be 128");
    if (c->d_model % 256) return set_error("mmdp_model_create: d_model must be a multiple of 256");
    if (c->mlp_hidden % 128) return set_error("mmdp_model_create: mlp_hidden must be a multiple of 128");
    if (c->vocab_size % 8) return set_error("mmdp_model_create: vocab_size must be a multiple of 8");
    if (c->n_layers <= 0 || c->max_seq_len <= 0 || c->max_batch <= 0) return set_error("mmdp_model_create: bad sizes");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return set_error("mmdp_model_create: no CUDA device (this library has no CPU fallback)");
    mmdp_model* m = new mmdp_model();
    m->cfg = *c;
    const size_t d = c->d_model, ff = c->mlp_hidden, V = c->vocab_size;
    m->layers.resize(c->n_layers);
    int rc = 0;
    for (auto& l : m->layers) {
        rc |= dev_alloc(m, (void**)&l.wqkv, 3 * d * d * 2);
        rc |= dev_alloc(m, (void**)&l.wo, d * d * 2);
        rc |= dev_alloc(m, (void**)&l.w13, 2 * ff * d * 2);
        rc |= dev_alloc(m, (void**)&l.w2, d * ff * 2);
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
    rc |= dev_alloc(m, (void**)&m->k, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->att, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->xr, Mm * d * 2);
    rc |= dev_alloc(m, (void**)&m->h, Mm * ff * 2);
    rc |= dev_alloc(m, (void**)&m->vt, (size_t)c->max_batch * d * m->Lpad_max * 2);
    rc |= dev_alloc(m, (void**)&m->cos_tab, (size_t)c->max_seq_len * 64 * 4);
    rc |= dev_alloc(m, (void**)&m->sin_tab, (size_t)c->max_seq_len * 64 * 4);
    rc |= dev_alloc(m, (void**)&m->err_flag, sizeof(int));
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

MMDP_API int mmdp_model_set_weight(mmdp_model* m, const char* name, const void* src, int64_t rows, int64_t cols, void* stream) {
    if (!m || !name || !src) return set_error("mmdp_model_set_weight: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t d = m->cfg.d_model, ff = m->cfg.mlp_hidden, V = m->cfg.vocab_size;
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
    if (!strcmp(sub, "q_proj") || !strcmp(sub, "k_proj") || !strcmp(sub, "v_proj")) {
        if (expect(d, d)) return -1;
        const int which = sub[0] == 'q' ? 0 : (sub[0] == 'k' ? 1 : 2);
        return copy_rows(l.wqkv + (size_t)which * d * d, src, d * d * 2, s);
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
    const int d = c.d_model, ff = c.mlp_hidden, V = c.vocab_size, H = c.n_heads;
    const int M = B * L;
    const int Lpad = ((L + 7) / 8) * 8;
    if (m->vt_Lpad != Lpad || L < m->vt_L) {  // (indexing depends on Lpad only; batch rows are disjoint)
        // pad columns [L, Lpad) of V^T must be zero (they meet P == 0 in the P·V MMA): re-zero when the layout changes or
        // when L shrinks inside the same Lpad (columns a longer forward wrote would otherwise stay behind)
        MMDP_CUDA(cudaMemsetAsync(m->vt, 0, (size_t)c.max_batch * d * m->Lpad_max * 2, s));
        m->vt_B = B;
        m->vt_Lpad = Lpad;
    }
    m->vt_L = L;
    const float scale = 1.0f / sqrtf(128.0f);
    if (embed_rows(ids, m->wte, m->x, M, d, V, s, m->err_flag)) return -1;
    QkvRopeArgs qa{m->q, m->k, m->vt, m->cos_tab, m->sin_tab, L, Lpad, d, H};
    // Row window of the LAST block: nothing after the last block mixes rows (ln_f and the LM head are row-wise and only the rows in
    // rows_a / rows_b are read), so its query rows / attn_out / MLP outside positions [row_lo, row_hi) of every batch row are dead
    // work: the keys and values of ALL rows are still computed, the rest of the block runs on the window only (per batch row).
    const bool window = !full_logits && opt(OPT_ROW_WINDOW) && row_hi > row_lo && row_lo >= 0 && row_hi <= L && (row_hi - row_lo) < L;  // MMDP_ROW_WINDOW=0: A/B switch
    if (!window) { row_lo = 0; row_hi = L; }
    for (int li = 0; li < c.n_layers; ++li) {
        const LayerWeights& l = m->layers[li];
        const bool win = window && li == c.n_layers - 1;
        if (rmsnorm(m->x, d, l.attn_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_QKVROPE, m->xn, d, l.wqkv, d, M, 3 * d, d, nullptr, 0, nullptr, 0, &qa, s)) return -1;
        if (!win) {
            if (attention_fwd(m->q, m->k, m->vt, m->att, B, H, L, Lpad, scale, s)) return -1;
            if (gemm_bf16(EPI_RESID, m->att, d, l.wo, d, M, d, d, m->x, d, m->x, d, nullptr, s)) return -1;
            if (rmsnorm(m->x, d, l.ff_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
            if (gemm_bf16(EPI_SWIGLU, m->xn, d, l.w13, d, M, 2 * ff, d, m->h, ff, nullptr, 0, nullptr, s)) return -1;
            if (gemm_bf16(EPI_RESID, m->h, ff, l.w2, ff, M, d, ff, m->x, d, m->x, d, nullptr, s)) return -1;
            continue;
        }
        const int Mw = row_hi - row_lo;
        for (int b = 0; b < B; ++b) {  // one row range per batch row (B = 1, or the CFG batch of variant M)
            const size_t r0 = (size_t)b * L + row_lo, o_d = r0 * d, o_ff = r0 * ff;
            if (attention_fwd(m->q + o_d, m->k + (size_t)b * L * d, m->vt + (size_t)b * H * 128 * Lpad, m->att + o_d, 1, H, L, Lpad, scale, s, Mw)) return -1;
            if (gemm_bf16(EPI_RESID, m->att + o_d, d, l.wo, d, Mw, d, d, m->x + o_d, d, m->x + o_d, d, nullptr, s)) return -1;
            if (rmsnorm(m->x + o_d, d, l.ff_norm, m->xn + o_d, d, Mw, d, c.rms_eps, s)) return -1;
            if (gemm_bf16(EPI_SWIGLU, m->xn + o_d, d, l.w13, d, Mw, 2 * ff, d, m->h + o_ff, ff, nullptr, 0, nullptr, s)) return -1;
            if (gemm_bf16(EPI_RESID, m->h + o_ff, ff, l.w2, ff, Mw, d, ff, m->x + o_d, d, m->x + o_d, d, nullptr, s)) return -1;
        }
    }
    if (full_logits) {
        if (rmsnorm(m->x, d, m->ln_f, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_PLAIN, m->xn, d, m->head, d, M, V, d, (bf16*)full_logits, V, nullptr, 0, nullptr, s)) return -1;
    }
    if (n_a > 0) {
        if (!rows_a || !out_a) return set_error("mmdp_model_forward: rows_a/out_a null");
        if (n_a > m->Mmax) return set_error("mmdp_model_forward: too many rows_a");
        if (rmsnorm_rows(m->x, d, rows_a, m->ln_f, m->xr, d, n_a, d, c.rms_eps, s, M, m->err_flag, window ? row_lo : 0, window ? row_hi : 0, window ? L : 0)) return -1;
        if (gemm_bf16(EPI_PLAIN, m->xr, d, m->head, d, n_a, V, d, (bf16*)out_a, V, nullptr, 0, nullptr, s)) return -1;
    }
    if (n_b > 0) {
        if (!rows_b || !out_b) return set_error("mmdp_model_forward: rows_b/out_b null");
        if (n_a + n_b > m->Mmax) return set_error("mmdp_model_forward: too many rows_a + rows_b");
        bf16* xr_b = m->xr + (size_t)n_a * d;
        if (rmsnorm_rows(m->x, d, rows_b, m->ln_f, xr_b, d, n_b, d, c.rms_eps, s, M, m->err_flag, window ? row_lo : 0, window ? row_hi : 0, window ? L : 0)) return -1;
        if (gemm_bf16(EPI_PLAIN, xr_b, d, m->head + (size_t)col0_b * d, d, n_b, ncols_b, d, (bf16*)out_b, ncols_b, nullptr, 0, nullptr, s)) return -1;
    }
    return 0;
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

MMDP_API int mmdp_model_forward_cached(mmdp_model* m, const int64_t* ids, int B, int L, int Tq, const int32_t* pos_map, uint16_t* kcache,
                              uint16_t* vtcache, uint16_t* logits, void* stream) {
    if (!m || !ids || !kcache || !vtcache) return set_error("mmdp_model_forward_cached: null argument");
    const mmdp_model_config& c = m->cfg;
    if (B <= 0 || B > c.max_batch || L <= 0 || L > c.max_seq_len || Tq <= 0 || Tq > L)
        return set_error("mmdp_model_forward_cached: B=%d L=%d Tq=%d outside workspace (max_batch=%d max_seq_len=%d)", B, L, Tq, c.max_batch, c.max_seq_len);
    if (!pos_map && Tq != L) return set_error("mmdp_model_forward_cached: a partial forward needs the position map");
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
        if (gemm_bf16(EPI_QKVROPE, m->xn, d, l.wqkv, d, M, 3 * d, d, nullptr, 0, nullptr, 0, &qa, s)) return -1;
        if (attention_fwd(m->q, kc, vc, m->att, B, H, L, Lpad, scale, s, Tq)) return -1;
        if (gemm_bf16(EPI_RESID, m->att, d, l.wo, d, M, d, d, m->x, d, m->x, d, nullptr, s)) return -1;
        if (rmsnorm(m->x, d, l.ff_norm, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_SWIGLU, m->xn, d, l.w13, d, M, 2 * ff, d, m->h, ff, nullptr, 0, nullptr, s)) return -1;
        if (gemm_bf16(EPI_RESID, m->h, ff, l.w2, ff, M, d, ff, m->x, d, m->x, d, nullptr, s)) return -1;
    }
    if (logits) {
        if (rmsnorm(m->x, d, m->ln_f, m->xn, d, M, d, c.rms_eps, s)) return -1;
        if (gemm_bf16(EPI_PLAIN, m->xn, d, m->head, d, M, V, d, (bf16*)logits, V, nullptr, 0, nullptr, s)) return -1;
    }
    return 0;
}

}  // extern "C"
