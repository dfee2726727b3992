/*
 * mmdp.h - C ABI of the H100-native (sm_90a) MMaDA-Parallel denoising hot path (libmmdp.so).
 *
 * The reference (tyfeld/MMaDA-Parallel) has no FFI/plugin layer: its boundary is the Python API
 *   generate_ti2ti(...)                         MMaDA-Parallel-A/generators/parallel_generator.py:102-368
 *   model(input_ids, infer=True).logits         MMaDA-Parallel-A/model/modeling_xllmx_dimoo.py:41-72
 *   MMadaModelLM.interleave_generate(...)       MMaDA-Parallel-M/models/modeling_mmada.py:118-248
 *   MAGVITv2.decode_code(...)                   MMaDA-Parallel-M/models/modeling_magvitv2.py:429-433
 * Every entry point below is what a ctypes stub under those callables binds (see INTEGRATION.md); each comment
 * names the reference lines the call replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host; bf16 tensors are passed as uint16_t*;
 *   - every function returns 0 on success, -1 on failure; mmdp_last_error() returns the (thread-local) message;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); no call synchronises the device;
 *   - nothing here falls back to the CPU: without a CUDA device every compute call fails with an error.
 */
#ifndef MMDP_H_
#define MMDP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMDP_VERSION 100
#if defined(__GNUC__)
#define MMDP_API __attribute__((visibility("default")))
#else
#define MMDP_API
#endif

MMDP_API int mmdp_version(void);
MMDP_API const char* mmdp_last_error(void);

/* ---- launch accounting (bench.py: gpu_launches and the live roofline pass) ------------------------------------------
 * kinds: 0 = GEMM (work = flops), 1 = attention (flops), 2 = row kernels embed/rmsnorm/lfq (bytes), 3 = sampling (bytes).
 * mmdp_prof_enable(1) brackets every subsequent launch with CUDA events on its stream; mmdp_prof_summary synchronises
 * and returns, per kind, summed milliseconds / algorithmic work / launch count (arrays of 4). */
MMDP_API void mmdp_prof_enable(int on);
MMDP_API int mmdp_prof_summary(double* ms, double* work, long long* launches);
MMDP_API long long mmdp_launch_count(int reset);
/* Kernel selection for GEMMs: 0 (default) = one CTA per 128xN tile (with its split-K tail), 1 = for M > 256 a cluster of two
 * CTAs per pair of m-adjacent 128xN tiles, the W tile multicast to both (TMA multicast), 2 = pairs only for M >= 4096 and
 * N >= 8192. Without the split-K tail the two kernels are bit-identical (same K order); also MMDP_GEMM_PAIR. */
MMDP_API void mmdp_set_gemm_pair(int on);
/* Split-K tail of the persistent GEMM (csrc/gemm.cu): 0 = never, 1 = residual epilogues only, 2 (default) = every epilogue
 * where the launch planner's cost model says it pays, 3 = whenever a partial last wave exists (tests).
 * The tiles of a partial last wave are split along K over the idle SMs; partial sums meet in an fp32 workspace owned per
 * (device, stream) and are reduced in fixed split order, so results are deterministic for a given (M, N, K) but the fp32
 * summation order of those tiles differs from the unsplit kernel (same bf16 rounding points). Such launches are
 * cooperative (co-residency of the grid is guaranteed by the runtime). Also MMDP_GEMM_SPLITK. */
MMDP_API void mmdp_set_gemm_splitk(int mode);
/* Programmatic dependent launch between the kernels of a forward (1 = default): a kernel's prologue (barrier init,
 * descriptor prefetch) overlaps the tail of its predecessor; every kernel waits for the
 * predecessor's completion (griddepcontrol.wait) before touching its data. Also MMDP_PDL=0|1. */
MMDP_API void mmdp_set_pdl(int on);
/* Generic tuning knob (bench/profiling tools): keys "pdl", "gemm_splitk", "gemm_l2pf" (L2 prefetch distance of weight tiles
 * in k-blocks, 0 = off), "gemm_l2pf_mod", "gemm_pair", "gemm_group_m", "attn_split_tail" (KV-split of attention's
 * partial last wave), "attn_version" (6: 128-key blocks, 7: 64-key blocks), "rmsnorm_warp", "row_window". Each defaults to the environment variable MMDP_<KEY in upper case>. */
MMDP_API int mmdp_set_option(const char* key, int value);

/* ---- tensor-parallel collective over NVLink peer memory (BASELINE config 4; csrc/tp_collective.cu) --------------------------
 * The reference has no tensor parallelism; this replaces what an nn.Module sharded over GPUs would do with NCCL after the two
 * row-parallel linears of a block (attn_out modeling_llada.py:744, ff_out :968): all-reduce, residual add (:953/:970) and the
 * next RMSLayerNorm (:315-329): the GEMM epilogue pushes each fp32 partial row to the rank that owns it (the reduce-scatter,
 * overlapped with the GEMM's main loop), then ONE kernel per rank sums the rows IT OWNS (fixed rank order), applies
 * x = bf16(bf16(sum) + x) and the norm, and stores the bf16 result into every rank's activation buffer (P2P stores, the
 * all-gather). Flags with a monotonically increasing
 * `epoch` synchronise the ranks; the call also enqueues the wait for all ranks' rows, so the next kernel on `stream` may read xn.
 *   mmdp_tp_alloc / mmdp_tp_free      zeroed device buffer suitable for IPC export (a plain cudaMalloc)
 *   mmdp_ipc_export / _import / _close 64-byte CUDA IPC handle of a buffer / peer mapping of another rank's buffer (same node)
 *   mmdp_gemm_f32_scatter             C = A W^T in fp32, each row PUSHED from the epilogue into the receive buffer of the rank that
 *                                     owns it: recv[row / rows_per_rank] + (slot * rows_per_rank + row % rows_per_rank) * N
 *                                     (recv: HOST array of n_ranks peer-mapped buffers [n_ranks][rows_per_rank][N] fp32; slot = this
 *                                     rank). The reduce-scatter of the row-parallel linears, fused into the GEMM.
 *   recv_local                        this rank's receive buffer (slot r = rank r's partial rows for the rows this rank owns)
 *   xn[r], flags[r]                   HOST arrays of n_ranks device pointers: rank r's activation buffer [M, d] bf16 and flag
 *                                     array [2][8] uint32 (own buffers for r == my_rank, imported mappings otherwise).
 *                                     n_src = n_ranks, or 0 = no partial sums (norm + broadcast only).
 *   x_shard [nrows, d] bf16           this rank's rows [row0, row0 + nrows) of the residual stream (updated in place)
 *   done_counter                      one zeroed uint32 in device memory. Two receive buffers must be used alternately. */
MMDP_API int mmdp_tp_alloc(uint64_t bytes, void** out);
MMDP_API int mmdp_tp_free(void* p);
MMDP_API int mmdp_ipc_export(void* p, uint8_t* handle64);
MMDP_API int mmdp_ipc_import(const uint8_t* handle64, void** out);
MMDP_API int mmdp_ipc_close(void* p);
MMDP_API int mmdp_gemm_f32_scatter(const uint16_t* A, int lda, const uint16_t* W, int ldw, int M, int N, int K, float* const* recv,
                          int n_ranks, int rows_per_rank, int slot, void* stream);
MMDP_API int mmdp_tp_reduce_norm(const float* recv_local, int rows_per_rank, int n_src, uint16_t* const* xn, uint32_t* const* flags,
                        int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* weight, int row0, int nrows, int d, float eps,
                        uint32_t epoch, uint32_t* done_counter, void* stream);

/* The whole tensor-parallel body in one call (the per-layer sequence TensorParallelLLaDA used to issue from Python: ~10 launches
 * per layer left a TP=8 rank CPU-bound): embedding of this rank's rows, norm + broadcast, then per layer column-parallel QKV+RoPE,
 * attention on the local heads, row-parallel attn_out pushed to the owners, reduce + residual + ff_norm + broadcast, column-parallel
 * gate/up + SwiGLU, row-parallel ff_out pushed, reduce + residual + next norm (ln_f after the last layer) + broadcast.
 * On return (stream order) every rank's xn buffer holds ln_f(x) for all B*L rows. Pointers are device pointers owned by the caller. */
typedef struct mmdp_tp_layer {
    const uint16_t* wqkv;       /* [3 * d_attn, d]  q | k | v rows of the local heads */
    const uint16_t* wo;         /* [d, d_attn] */
    const uint16_t* w13;        /* [2 * ff_local, d] gate / up interleaved in 128-row blocks */
    const uint16_t* w2;         /* [d, ff_local] */
    const uint16_t* attn_norm;  /* [d] */
    const uint16_t* ff_norm;    /* [d] */
} mmdp_tp_layer;
/* Shared (peer-mapped) state of one ROW CHUNK of the tensor-parallel forward. The sequence rows are cut into n_chunks (1 or 2)
 * contiguous chunks; inside a chunk rank r owns rows [r*R, (r+1)*R), R = ceil(rows of the chunk / n_ranks). With two chunks
 * the attn_out / MLP part of a layer runs as two independent chains on two streams, so that one chunk's NVLink traffic
 * (partial rows pushed from the GEMM epilogue, broadcast of the normalised rows) overlaps the other chunk's GEMMs. */
typedef struct mmdp_tp_chunk {
    uint16_t* x_shard;                           /* this rank's rows of the residual stream [R, d] */
    float* const* recv[2];                       /* HOST arrays [n_ranks] of the two receive buffers of every rank ([n_ranks][R][d] fp32 each) */
    uint32_t* const* flags;                      /* HOST array [n_ranks] of the flag arrays ([2][8] uint32 each) */
    uint32_t* done_counter;
} mmdp_tp_chunk;
typedef struct mmdp_tp_ctx {
    int32_t d_model, n_heads_local, ff_local, n_layers, n_ranks, rank;
    float rms_eps;
    const mmdp_tp_layer* layers;                 /* HOST array [n_layers] */
    const uint16_t* wte; const uint16_t* ln_f; int64_t vocab;
    const float* cos_tab; const float* sin_tab;  /* [max_seq_len, 64] */
    uint16_t *q, *k, *att, *h, *vt;              /* work buffers: [M, d_attn] x3, [M, ff_local], [B, H_local, 128, Lpad] (pad columns zero) */
    uint16_t* const* xn;                         /* HOST array [n_ranks] of the activation buffers [M, d] */
    int32_t n_chunks;                            /* 1 or 2 */
    int32_t chunk_rows0;                         /* rows of chunk 0 (chunk 1 holds the rest); ignored when n_chunks == 1 */
    mmdp_tp_chunk chunk[2];
} mmdp_tp_ctx;
/* epoch0: the last epoch used so far; the call uses epoch0 + 1 ... epoch0 + 2 * n_layers + 1 on every chunk's flags (returned
 * through *epoch_out). With two chunks the call uses an internal second stream, forked from and joined back into `stream`. */
MMDP_API int mmdp_tp_forward(const mmdp_tp_ctx* c, const int64_t* ids, int B, int L, uint32_t epoch0, uint32_t* epoch_out, void* stream);

/* ---- epilogues of mmdp_gemm_bf16 ----------------------------------------------------------------------------- */
#define MMDP_EPI_PLAIN 0   /* C = bf16(A W^T)                                 nn.Linear, modeling_llada.py:1402      */
#define MMDP_EPI_RESID 1   /* C = bf16(bf16(A W^T) + R)                       attn_out :744 + :953; ff_out :968+:970  */
#define MMDP_EPI_F32 4     /* C (float*) = raw fp32 accumulators: tensor-parallel partial sums, all-reduced before rounding      */
#define MMDP_EPI_SWIGLU 3  /* C = bf16(bf16(silu(bf16 g)) * bf16 u), W rows interleaved 128 gate / 128 up   :962-967 */

/* C[M,N] = A[M,K] * W[N,K]^T, bf16 in, fp32 accumulate (wgmma), fused epilogue.
 * lda/ldw/ldc/ldr are row strides in elements (multiples of 8). For MMDP_EPI_SWIGLU, C has N/2 columns. */
MMDP_API int mmdp_gemm_bf16(int epilogue, const uint16_t* A, int lda, const uint16_t* W, int ldw, int M, int N, int K,
                   uint16_t* C, int ldc, const uint16_t* R, int ldr, void* stream);

/* q/k/v projection + rotary embedding (modeling_llada.py:925-927, RotaryEmbedding :402-435).
 * Wqkv = [q_proj; k_proj; v_proj] rows ([3*d_model, d_model]); A = normed activations [B*L, d_model].
 * Outputs: q,k [B*L, d_model] with RoPE applied (fp32 math on the bf16-rounded projections, positions 0..L-1 per batch row);
 * vt [B, n_heads, 128, Lpad] = V transposed (token index contiguous); columns >= L of vt must be zero (never written).
 * cos/sin: fp32 [L, 64] tables (first half of the reference's cat(freqs, freqs) table). head_dim must be 128. */
MMDP_API int mmdp_qkv_rope(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads, int L, int Lpad,
                  const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream);

/* Tensor-parallel shard of the same projection: Wqkv = [q rows | k rows | v rows] of this rank's n_heads_local heads
 * ([3*128*n_heads_local, d_model]); q,k: [B*L, 128*n_heads_local]; vt: [B, n_heads_local, 128, Lpad]. */
MMDP_API int mmdp_qkv_rope_tp(const uint16_t* A, int lda, const uint16_t* Wqkv, int M, int d_model, int n_heads_local, int L,
                      int Lpad, const float* cos_tab, const float* sin_tab, uint16_t* q, uint16_t* k, uint16_t* vt, void* stream);

/* x = bf16(bf16(partial) + x): residual add of an fp32 partial-sum buffer that was all-reduced across tensor-parallel ranks
 * (keeps the reference's rounding points: nn.Linear output -> bf16, then the residual add -> bf16). */
MMDP_API int mmdp_resid_add_f32(uint16_t* x, int ldx, const float* partial, int ldp, int M, int d, void* stream);

/* softmax(q k^T * scale) v, no mask, non-causal (F.scaled_dot_product_attention call at modeling_llada.py:672-679).
 * q,k: [B*L, n_heads*128]; vt: [B, n_heads, 128, Lpad]; out: [B*L, n_heads*128]. Lpad >= L, Lpad % 8 == 0; the pad
 * columns vt[..., L:Lpad] must hold finite values (mmdp_qkv_rope leaves them untouched, mmdp_model_* keeps them zero):
 * they are multiplied by probabilities that are exactly or nearly (2^-126) zero. */
MMDP_API int mmdp_attention(const uint16_t* q, const uint16_t* k, const uint16_t* vt, uint16_t* out, int B, int n_heads, int L,
                   int Lpad, float scale, void* stream);

/* RMSLayerNorm.forward (modeling_llada.py:315-329). rows (nullable int32[M]) gathers input rows. */
MMDP_API int mmdp_rmsnorm(const uint16_t* x, int ldx, const int32_t* rows, const uint16_t* weight, uint16_t* y, int ldy, int M,
                 int d, float eps, void* stream);

/* wte lookup (modeling_llada.py:1265): x[i,:] = wte[ids[i],:] */
MMDP_API int mmdp_embed(const int64_t* ids, const uint16_t* wte, uint16_t* x, int M, int d, int64_t vocab, void* stream);

/* ---- mask-predict step --------------------------------------------------------------------------------------- */

/* Text step (parallel_generator.py:181-217; M: modeling_mmada.py:179-209).
 * cond/uncond: logits rows of the R text positions ([R, ld] bf16). uncond nullable (A); with uncond the logits are
 * cond + text_cfg*(uncond-cond) in bf16 (M). unoise nullable: torch.rand(dtype=bf16) noise [R, ld_noise] for A's
 * add_gumbel_noise at `temperature` > 0. ids_text points at the R ids of the text span inside the sequence; the k
 * most confident masked positions (fp64 softmax probability of the argmax token) are committed in place.
 * x0_ws int64[R], conf_ws double[R] are caller-provided workspaces (also the debug outputs). */
MMDP_API int mmdp_text_step(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int R, int V, float text_cfg,
                   const uint16_t* unoise, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
                   int k, int64_t* x0_ws, double* conf_ws, void* stream);

/* Image step (parallel_generator.py:220-344 for variant 0 = A; modeling_mmada.py:211-241 for variant 1 = M).
 * cond/unc_a/unc_b: [N, ld] bf16 logits restricted to the C codebook columns.
 *   A: logits = cond + s_a*(cond-unc_a) + s_b*(cond-unc_b)   (unc_a = uncond_text, unc_b = uncond_image; nullable)
 *   M: logits = s_b*cond - s_a*unc_a                           (caller passes s_b = 1+image_cfg, s_a = image_cfg)
 * qnoise nullable: Exp(1) noise [N, C] bf16 = the `q` torch.multinomial draws; null -> argmax(probs) (temperature 0).
 * conf_noise nullable [N] bf16: A randn / M uniform noise of mask_by_random_topk; temp = temperature*(1-ratio).
 * sched_len = floor(N * noise_schedule(ratio)) evaluated by the host exactly like the reference (fp32 torch scalar).
 * ids: full sequence id buffer (int64) updated in place at positions pos[0..N); vq_offset = text vocab size.
 * Workspaces/outputs: sampled_ws int32[N] (ids before re-masking = M's return value), selp_ws float[N],
 * unknown_ws uint8[N]; probs_out (nullable, [N, C] bf16), mask_len_out (nullable int32), masking_out (nullable uint8[N]). */
MMDP_API int mmdp_image_step(int variant, const uint16_t* cond, const uint16_t* unc_a, const uint16_t* unc_b, int64_t ld, int N,
                    int C, float s_a, float s_b, const uint16_t* qnoise, const uint16_t* conf_noise, float temp,
                    int sched_len, int64_t* ids, const int32_t* pos, int64_t mask_id, int64_t vq_offset,
                    int32_t* sampled_ws, float* selp_ws, uint8_t* unknown_ws, uint16_t* probs_out,
                    int32_t* mask_len_out, uint8_t* masking_out, void* stream);

/* Second half of the image step on its own (mask_by_random_topk + write-back): parallel_generator.py:23-70, :318-344;
 * M/models/sampling.py:31-36. Inputs are the per-token outputs of the first half (sampled ids, selected probabilities
 * as bf16-representable floats, unknown flags). Ties between equal confidences keep the lower index masked first. */
/* Text step with variant M's fp64 Gumbel-max (M/models/modeling_mmada.py:49-60 `add_gumbel_noise`, used at :185 and :659 when
 * the text temperature is > 0): x0 = argmax_v exp(double(l_v)) / (-log u_v)^temperature with u = unoise64 [R, ld_noise] fp64
 * uniform noise drawn by the caller exactly as the reference draws it (torch.rand_like(logits, dtype=float64), global RNG of
 * the logits' device). Everything else as mmdp_text_step. */
MMDP_API int mmdp_text_step_gumbel64(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int R, int V, float text_cfg,
                            const double* unoise64, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
                            int k, int64_t* x0_ws, double* conf_ws, void* stream);
/* One step of A's MaskGit text-to-image decoding, generate_image (MMaDA-Parallel-A/generators/image_generation_generator.py:
 * 119-208) on the N currently masked positions pos[0..N) of `ids` (compacted by the caller; every ids[pos[i]] == mask_id):
 *   logits = cond | (1 + cfg) * cond - cfg * uncond            (:156 / :162; uncond nullable, rows [N, C], bf16 at every op)
 *   sample = argmax(logits / tau + g(gumbel_u))  | argmax(logits) when gumbel_u is NULL (tau == 0)   (generation_utils.py:37-42)
 *   conf   = softmax(logits)[sample] (bf16)                                                          (:173-174)
 *   ids[pos] = sample + vq_offset; then positions with log(clamp_min(conf,1e-20)) + temperature * g(conf_u) strictly below the
 *   keep_n-th smallest (keep_n clamped to [0, N-1]) are set back to mask_id                          (generation_utils.py:45-61)
 * g(u) = -log(-log(u + 1e-20) + 1e-20) in bf16. Workspaces: sampled_ws int32 [N], selp_ws float [N], unknown_ws uint8 [N];
 * masking_out (nullable) uint8 [N]. */
MMDP_API int mmdp_image_step_t2i(const uint16_t* cond, const uint16_t* uncond, int64_t ld, int N, int C, float cfg,
                        const uint16_t* gumbel_u, float tau, const uint16_t* conf_u, float temperature, int keep_n,
                        int64_t* ids, const int32_t* pos, int64_t mask_id, int64_t vq_offset, int32_t* sampled_ws,
                        float* selp_ws, uint8_t* unknown_ws, uint8_t* masking_out, void* stream);
MMDP_API int mmdp_image_remask(int variant, int N, const int32_t* sampled, const float* selp, const uint8_t* unknown,
                      const uint16_t* conf_noise, float temp, int sched_len, int64_t* ids, const int32_t* pos,
                      int64_t mask_id, int64_t vq_offset, int32_t* mask_len_out, uint8_t* masking_out, void* stream);

/* LFQuantizer.get_codebook_entry (modeling_magvitv2.py:208-221): ids [B, N] -> z_q fp32 [B, bits, N] (+-1). */
MMDP_API int mmdp_lfq_decode(const int64_t* ids, float* zq, int B, int N, int bits, void* stream);

/* ---- VQ decoder context: MAGVITv2.decode_code (M/models/modeling_magvitv2.py:429-433, VQGANDecoder :278-399) -------- */
typedef struct mmdp_vqdec mmdp_vqdec;
typedef struct {
    int32_t ch;                 /* 128 */
    int32_t n_levels;           /* len(ch_mult), <= 8 */
    int32_t ch_mult[8];         /* (1, 1, 2, 2, 4) */
    int32_t num_res_blocks[8];  /* (4, 4, 3, 4, 3) */
    int32_t z_channels;         /* 13 = LFQ bits */
    int32_t out_ch;             /* 3 */
    int32_t max_batch;
    int32_t latent_h, latent_w; /* 32 x 32 code grid -> 512 x 512 pixels */
} mmdp_vqdec_config;

MMDP_API int mmdp_vqdec_create(const mmdp_vqdec_config* cfg, mmdp_vqdec** out);
MMDP_API void mmdp_vqdec_destroy(mmdp_vqdec* d);
/* name = reference parameter name ("decoder.conv_in.weight", "decoder.up.3.block.0.norm1.bias", ...); src = fp32, device or
 * host pointer, reference layout (conv: OIHW). Convolution weights are repacked to the tap-major layout of the TF32 GEMM. */
MMDP_API int mmdp_vqdec_set_weight(mmdp_vqdec* d, const char* name, const float* src, int64_t numel, void* stream);
/* number of parameters not loaded yet (names written space-separated into out, truncated to out_len) */
MMDP_API int mmdp_vqdec_missing(mmdp_vqdec* d, char* out, int out_len);
/* ids int64 [B, h*w] (device) -> pixels fp32 [B, out_ch, H, W] (device), H = h * 2^(n_levels-1). */
MMDP_API int mmdp_vqdec_decode(mmdp_vqdec* d, const int64_t* ids, int B, int h, int w, float* out_nchw, void* stream);

/* VQ encoder context: MAGVITv2.get_code (modeling_magvitv2.py:423-427). Same config struct (out_ch = image channels,
 * latent_h/w = code grid => pixels = latent << (n_levels-1); ch_mult / num_res_blocks in ENCODER order (1,2,2,4,4)/(4,3,4,3,4));
 * parameters are loaded with mmdp_vqdec_set_weight under the reference's 'encoder.*' names; destroy with mmdp_vqdec_destroy.
 * pixels fp32 [B, 3, H, W] (device) -> ids int64 [B, (H/16)*(W/16)]. */
MMDP_API int mmdp_vqenc_create(const mmdp_vqdec_config* cfg, mmdp_vqdec** out);
MMDP_API int mmdp_vqenc_encode(mmdp_vqdec* enc, const float* pixels_nchw, int B, int H, int W, int64_t* ids_out, void* stream);

/* ---- whole-model context (LLaDAModel.forward, modeling_llada.py:1201-1415) ----------------------------------- */
typedef struct mmdp_model mmdp_model;

typedef struct {
    int32_t d_model;      /* 4096 */
    int32_t n_heads;      /* 32, head_dim must be 128 */
    int32_t n_layers;     /* 32 */
    int32_t mlp_hidden;   /* 12288 = rows of ff_proj / up_proj */
    int32_t vocab_size;   /* rows of wte and of the LM head (embedding_size) */
    int32_t max_seq_len;  /* workspace sizing */
    int32_t max_batch;    /* workspace sizing (CFG batch) */
    float rms_eps;
} mmdp_model_config;

MMDP_API int mmdp_model_create(const mmdp_model_config* cfg, mmdp_model** out);
MMDP_API void mmdp_model_destroy(mmdp_model* m);

/* Copies (and packs) one tensor of the HF state dict into the model-owned device buffers. `src` may be a device or
 * a pinned/pageable host pointer (cudaMemcpyDefault). Names (layer = 0..n_layers-1):
 *   "wte" [V,d], "ln_f" [d], "head" [V,d],
 *   "blocks.<i>.q_proj|k_proj|v_proj|attn_out" [d,d], "blocks.<i>.ff_proj|up_proj" [ff,d], "blocks.<i>.ff_out" [d,ff],
 *   "blocks.<i>.attn_norm|ff_norm" [d]. */
MMDP_API int mmdp_model_set_weight(mmdp_model* m, const char* name, const void* src, int64_t rows, int64_t cols, void* stream);

/* fp32 rotary tables [L, 64] (cos, sin), computed by the host exactly like RotaryEmbedding.get_rotary_embedding. */
MMDP_API int mmdp_model_set_rope(mmdp_model* m, const float* cos_tab, const float* sin_tab, int L, void* stream);

/* One forward over ids [B, L]. Logits are produced only where requested:
 *   full_logits   (nullable) [B*L, V]                      - the reference contract (model(...).logits)
 *   rows_a/out_a  (nullable) n_a flattened row indices (b*L + pos) x all V columns      -> out_a [n_a, V]
 *   rows_b/out_b  (nullable) n_b flattened row indices x columns [col0_b, col0_b+ncols_b) -> out_b [n_b, ncols_b] */
MMDP_API int mmdp_model_forward(mmdp_model* m, const int64_t* ids, int B, int L, uint16_t* full_logits, const int32_t* rows_a,
                       int n_a, uint16_t* out_a, const int32_t* rows_b, int n_b, int col0_b, int ncols_b,
                       uint16_t* out_b, void* stream);
/* The same with a ROW WINDOW for the last block (rows_a / rows_b only): nothing after the last block mixes rows, so only rows that
 * are read (every index of rows_a / rows_b must be a position in [row_lo, row_hi) of its batch row: (index % L) inside the window)
 * need its attention output and MLP; keys and values of all rows are still computed; one launch set per batch row. Output-invariant dead-work elimination (identical GEMM results per row; the attention rows differ
 * from the unwindowed launch only by which query tiles take the KV-split path). A row index outside the window raises bit 2 of the
 * error flags (mmdp_model_error_flags). row_hi <= row_lo disables the window. */
MMDP_API int mmdp_model_forward_window(mmdp_model* m, const int64_t* ids, int B, int L, const int32_t* rows_a, int n_a, uint16_t* out_a,
                              const int32_t* rows_b, int n_b, int col0_b, int ncols_b, uint16_t* out_b, int row_lo, int row_hi,
                              void* stream);

/* Debug/testing: copy of the residual stream after `layer` layers is kept when enabled (device pointer returned). */
MMDP_API const uint16_t* mmdp_model_hidden(mmdp_model* m);
/* Token-cache forward: LLaDAModelLM.forward(input_ids, use_cache=True, to_compute_mask=mask, cat=key)
 * (MMaDA-Parallel-A/model/modeling_llada.py:1244-1245, :929-940, :715-716, :1406-1413). Computes the Tq selected tokens of every
 * batch row against the FULL cached key / value set and refreshes the caches at their positions first:
 *   ids [B*Tq] ids of the selected tokens (batch-row major); pos_map [B*Tq] their sequence positions (int32), or NULL with
 *   Tq == L for a full forward that fills the caches; kcache [n_layers][B*L][d] bf16 (keys after rotary); vtcache
 *   [n_layers][B][H][128][Lpad] bf16 (values transposed, Lpad = L rounded up to 8, pad columns zero - allocate zeroed);
 *   logits (nullable) [B*Tq][V] bf16 of the selected tokens. The caches are owned by the caller, one set per `cat` key. */
MMDP_API int mmdp_model_forward_cached(mmdp_model* m, const int64_t* ids, int B, int L, int Tq, const int32_t* pos_map, uint16_t* kcache,
                              uint16_t* vtcache, uint16_t* logits, void* stream);
/* Sticky device-side error flags of the forwards issued so far, read and cleared (this call SYNCHRONISES `stream`):
 * bit 0 = a token id was outside [0, vocab_size) (torch raises IndexError in nn.Embedding; the kernel read row 0),
 * bit 1 = a logits row index (rows_a / rows_b) was outside [0, B*L). The host mirrors call it at their read-back point. */
MMDP_API int mmdp_model_error_flags(mmdp_model* m, int32_t* flags_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMDP_H_ */
