// Fused epilogues of the bf16 GEMM kernel (gemm.cu) and the e4m3 GEMM kernel (fp8.cu). gemm_epilogue_tile handles one thread's
// wgmma fragment of a 128 x BN accumulator tile held in registers; epi_row8 handles one (row, 8-column) item for the split-K
// finishing pass and the staged epilogue of gemm_bf16_kernel.
#pragma once
#include "mmdp_internal.h"
#include "ptx.cuh"

namespace mmdp {

struct GemmParams {
    int M, N, K;
    __nv_bfloat16* C;
    int ldc;
    const __nv_bfloat16* resid;
    int ldr;
    // EPI_QKVROPE
    __nv_bfloat16* q;
    __nv_bfloat16* k;
    __nv_bfloat16* vt;
    const float* cos_tab;  // [L, 64]
    const float* sin_tab;  // [L, 64]
    int L, Lpad, d_model, n_heads;
    // token-cache forward (modeling_llada.py:929-940): the GEMM rows are a COMPACT subset of the sequence - row r is token
    // pos_map[r] of batch row r / Tq; q stays compact, k / v^T are scattered into the per-layer cache at that position.
    // nullptr: row r is token r % L of batch row r / L
    const int* pos_map;
    int Tq;
    int row0;  // QKVROPE: sequence index of GEMM row 0 (row-chunked launches); q / k are addressed relative to it, positions and V^T absolutely
    // split-K tail (gemm.cu): the last `sk_tail` tiles (a partial wave) are split along K into `sk_splits` (<= 8) units of
    // `sk_kb_per` k-blocks; partial accumulators meet in `sk_ws` (fp32, [tail][splits][BN/4][128] float4: column-group major,
    // tile row minor, so that the finishing threads (consecutive threads = consecutive rows) read contiguous 16-byte
    // pieces), `sk_cnt[2*tile]` counts arrivals
    int sk_tail, sk_splits, sk_kb_per;
    float* sk_ws;
    int* sk_cnt;
    // L2 prefetch distance in k-blocks for the weight tiles (0 = off) and the share of CTAs issuing it (every l2pf_mod-th m-tile)
    int l2pf, l2pf_mod;
    // EPI_F32 scatter (tensor parallel, GEMM fused with the reduce-scatter): scat_R > 0 -> the fp32 partial row `row` is
    // not stored to C but PUSHED over NVLink into its owner's receive buffer, scat_dst[row / scat_R] (peer-mapped,
    // [n_ranks][scat_R][ldc] fp32), slot scat_slot = this rank
    float* scat_dst[8];
    int scat_R, scat_slot;
    // tile order: group_m == 0 -> M-fastest over all m-tiles; > 0 -> M-fastest inside groups of group_m m-tiles, all n-tiles
    // of a group before the next group (keeps the group's A rows L2-resident while the weights stream)
    int group_m;
    // EPI_QKVROPE_PACKED: (sequence, position) of every row of a packed variable-length batch; q / k stay at the row,
    // v^T goes to vt[sequence][head][d][position]
    const int2* seg_pos;
    // EPI_QKVGQA*: kv heads (k is [M, 128 n_kv_heads], v^T [B][n_kv_heads][128][Lpad]) and the q | k | v bias (nullable)
    int n_kv_heads;
    const __nv_bfloat16* bias;
};

// Host-side argument check of the grouped-query QKV epilogues (bf16 and e4m3 GEMM). The token-cache launch stays on the
// multi-head epilogue; a row-chunked launch (the tensor-parallel forward's second chunk) takes positions and V^T through row0
// as EPI_QKVROPE does (qkv_row_coords), q / k relative to the chunk.
inline int qkv_gqa_check(const char* who, int epi, int M, int N, const QkvRopeArgs* qa) {
    if (!qa) return set_error("%s: qkv epilogue needs QkvRopeArgs", who);
    const int d = qa->d_model, H = qa->n_heads, Hkv = qa->n_kv_heads;
    if (d % 256 || d != H * 128) return set_error("%s: qkv epilogue needs head_dim 128 and d_model %% 256 == 0", who);
    if (Hkv <= 0 || Hkv > H || H % Hkv) return set_error("%s: n_kv_heads=%d must divide n_heads=%d", who, Hkv, H);
    if (N != d + 2 * 128 * Hkv) return set_error("%s: grouped-query qkv needs N == d_model + 2 * 128 * n_kv_heads", who);
    if (qa->pos_map) return set_error("%s: grouped-query qkv has no token-cache form", who);
    if (qa->row0 < 0) return set_error("%s: row0 must not be negative", who);
    if (epi == EPI_QKVGQA_PACKED ? (!qa->seg_pos || qa->chunked || qa->row0) : (qa->L <= 0 || (!qa->chunked && M % qa->L)))
        return set_error("%s: qkv epilogue needs M == B*L (or a row chunk of it, or a packed row map)", who);
    return 0;
}

__host__ __device__ __forceinline__ void gemm_tile_coords(int tl, int num_m, int num_n, int group_m, int& m_blk, int& n_blk) {
    if (group_m <= 0 || group_m >= num_m) {
        m_blk = tl % num_m;
        n_blk = tl / num_m;
    } else {
        const int per_group = group_m * num_n;
        const int gid = tl / per_group, r = tl - gid * per_group;
        const int first = gid * group_m;
        const int gsz = (num_m - first < group_m) ? num_m - first : group_m;
        m_blk = first + r % gsz;
        n_blk = r / gsz;
    }
}

// Row and (sequence, position) of GEMM row `row` for the QKV epilogues (the same mapping as gemm_epilogue_tile's).
template <int EPI>
__device__ __forceinline__ void qkv_row_coords(const GemmParams& p, int row, int& b, int& pos) {
    if constexpr (epi_is_packed(EPI)) {
        const int2 sp = p.seg_pos[row];
        b = sp.x;
        pos = sp.y;
    } else if (p.pos_map) {
        b = row / p.Tq;
        pos = p.pos_map[row];
    } else {
        b = (row + p.row0) / p.L;
        pos = (row + p.row0) - b * p.L;
    }
}

// EPI_QKVGQA*: accumulator of GEMM column `col` plus its bias, in fp32 (nn.Linear rounds acc + bias to bf16 once)
__device__ __forceinline__ float qkv_biased(const GemmParams& p, int col, float acc) {
    return p.bias ? __fadd_rn(acc, __bfloat162float(p.bias[col])) : acc;
}

// EPI_QKVGQA*: the rotary pair (t1 at column c, t2 at c + 64 of a q / k head) and its two bf16 outputs, or a V^T element
__device__ __forceinline__ void rope_pair(float t1, float t2, float cs, float sn, float& a, float& b) {
    // (t * cos) + (rotate_half(t) * sin), fp32, no FMA contraction
    a = __fadd_rn(__fmul_rn(t1, cs), __fmul_rn(-t2, sn));
    b = __fadd_rn(__fmul_rn(t2, cs), __fmul_rn(t1, sn));
}

// EPI_QKVGQA*: destination of GEMM column `col` (a q / k head start + c, c < 64) of row `row`
__device__ __forceinline__ __nv_bfloat16* gqa_qk_dst(const GemmParams& p, int row, int col) {
    return col < p.d_model ? p.q + (size_t)row * p.d_model + col : p.k + (size_t)row * (p.n_kv_heads * 128) + (col - p.d_model);
}
// EPI_QKVGQA*: V^T element of GEMM column `col` (>= d + d_kv) for sequence b, position pos
__device__ __forceinline__ __nv_bfloat16* gqa_vt_dst(const GemmParams& p, int col, int b, int pos) {
    const int n = col - p.d_model - p.n_kv_heads * 128;
    return p.vt + ((size_t)(b * p.n_kv_heads + (n >> 7)) * 128 + (n & 127)) * p.Lpad + pos;
}

// One thread's share of a 128 x BN accumulator tile (gemm.cu): the wgmma fragment of its warpgroup's 64-row half,
// acc[4j + 2h + e] = tile row rit0 + 8h, tile column 8j + c0 + e (c0 = 2 * (lane % 4)). Every element goes through the
// same rounding points as the reference; only the mapping of elements to threads is the fragment's.
template <int EPI, int BN>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, const float (&acc)[BN / 2], int m_blk, int n_blk, int rit0,
                                                   int c0) {
    const int n0 = n_blk * BN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = m_blk * 128 + rit0 + 8 * h;
        if (row >= p.M) continue;
        if constexpr (EPI == EPI_F32) {
            // raw fp32 accumulators (tensor-parallel partial sums: reduced across ranks in fp32, rounded once afterwards);
            // scat_R > 0: the row is pushed to the receive buffer of the rank that owns it (fused reduce-scatter)
            float* dst;
            if (p.scat_R > 0) {
                const int owner = row / p.scat_R;
                dst = p.scat_dst[owner] + ((size_t)p.scat_slot * p.scat_R + (row - owner * p.scat_R)) * p.ldc;
            } else {
                dst = reinterpret_cast<float*>(p.C) + (size_t)row * p.ldc;
            }
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = n0 + 8 * j + c0;
                if (col < p.N) *reinterpret_cast<float2*>(dst + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        } else if constexpr (EPI == EPI_PLAIN || EPI == EPI_RESID) {
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = n0 + 8 * j + c0;
                if (col >= p.N) continue;
                const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
                uint32_t o;
                if constexpr (EPI == EPI_RESID) {
                    // nn.Linear output is rounded to bf16 first, then the residual add rounds again
                    const uint32_t rr = *reinterpret_cast<const uint32_t*>(p.resid + (size_t)row * p.ldr + col);
                    o = pack_bf16x2(__fadd_rn(bf16_lo(rr), bf16_round(a0)), __fadd_rn(bf16_hi(rr), bf16_round(a1)));
                } else {
                    o = pack_bf16x2(a0, a1);
                }
                *reinterpret_cast<uint32_t*>(p.C + (size_t)row * p.ldc + col) = o;
            }
        } else if constexpr (EPI == EPI_SWIGLU) {
            // tile columns [0,BN/2) = gate rows of W1, [BN/2,BN) = up rows of W3 (weights packed interleaved in BN/2-row blocks)
#pragma unroll
            for (int j = 0; j < BN / 16; ++j) {
                const int col = n_blk * (BN / 2) + 8 * j + c0;
                if (col >= p.N / 2) continue;
                float o[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float gg = bf16_round(acc[4 * j + 2 * h + e]);
                    const float uu = bf16_round(acc[4 * (j + BN / 16) + 2 * h + e]);
                    const float s = bf16_round(__fdiv_rn(gg, __fadd_rn(1.0f, expf(-gg))));  // silu -> bf16
                    o[e] = __fmul_rn(s, uu);
                }
                *reinterpret_cast<uint32_t*>(p.C + (size_t)row * p.ldc + col) = pack_bf16x2(o[0], o[1]);
            }
        } else if constexpr (EPI == EPI_QKVROPE || EPI == EPI_QKVROPE_PACKED) {
            const int region = n0 / p.d_model;  // 0 = Q, 1 = K, 2 = V (d_model % 256 == 0 is checked on the host)
            int b, pos;
            if constexpr (EPI == EPI_QKVROPE_PACKED) {
                const int2 sp = p.seg_pos[row];
                b = sp.x;
                pos = sp.y;
            } else if (p.pos_map) {
                b = row / p.Tq;
                pos = p.pos_map[row];
            } else {
                b = (row + p.row0) / p.L;
                pos = (row + p.row0) - b * p.L;
            }
            if (region < 2) {
                const size_t drow = (region == 0 || !p.pos_map) ? (size_t)row : (size_t)b * p.L + pos;  // k rows go to their sequence position
                __nv_bfloat16* dst = (region == 0 ? p.q : p.k) + drow * p.d_model + (n0 - region * p.d_model);
#pragma unroll
                for (int head = 0; head < BN / 128; ++head) {
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {  // columns c and c + 64 of the head: the rotary pair
                        const int j = head * 16 + jj, c = 8 * jj + c0;
                        const float2 cs = *reinterpret_cast<const float2*>(p.cos_tab + (size_t)pos * 64 + c);
                        const float2 sn = *reinterpret_cast<const float2*>(p.sin_tab + (size_t)pos * 64 + c);
                        const float csv[2] = {cs.x, cs.y}, snv[2] = {sn.x, sn.y};
                        float a[2], bb[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float t1 = bf16_round(acc[4 * j + 2 * h + e]);
                            const float t2 = bf16_round(acc[4 * (j + 8) + 2 * h + e]);
                            // (t * cos) + (rotate_half(t) * sin), fp32, no FMA contraction
                            a[e] = __fadd_rn(__fmul_rn(t1, csv[e]), __fmul_rn(-t2, snv[e]));
                            bb[e] = __fadd_rn(__fmul_rn(t2, csv[e]), __fmul_rn(t1, snv[e]));
                        }
                        *reinterpret_cast<uint32_t*>(dst + head * 128 + c) = pack_bf16x2(a[0], a[1]);
                        *reinterpret_cast<uint32_t*>(dst + head * 128 + 64 + c) = pack_bf16x2(bb[0], bb[1]);
                    }
                }
            } else {
                // V is written transposed: vt[b][head][d][token] so that P·V runs with both operands K-major
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int n = n0 - 2 * p.d_model + 8 * j + c0;
                    const int head = n >> 7, d0 = n & 127;
                    __nv_bfloat16* dst = p.vt + ((size_t)(b * p.n_heads + head) * 128 + d0) * p.Lpad + pos;
                    dst[0] = __float2bfloat16_rn(acc[4 * j + 2 * h]);
                    dst[p.Lpad] = __float2bfloat16_rn(acc[4 * j + 2 * h + 1]);
                }
            }
        } else if constexpr (epi_is_gqa(EPI)) {
            // q | k | v regions are 128-column aligned but a tile may straddle the k | v boundary: decided per head
            int b, pos;
            qkv_row_coords<EPI>(p, row, b, pos);
#pragma unroll
            for (int head = 0; head < BN / 128; ++head) {
                const int col0 = n0 + head * 128;
                if (col0 >= p.N) continue;
                if (col0 < p.d_model + p.n_kv_heads * 128) {
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int j = head * 16 + jj, c = 8 * jj + c0;
                        const float2 cs = *reinterpret_cast<const float2*>(p.cos_tab + (size_t)pos * 64 + c);
                        const float2 sn = *reinterpret_cast<const float2*>(p.sin_tab + (size_t)pos * 64 + c);
                        const float csv[2] = {cs.x, cs.y}, snv[2] = {sn.x, sn.y};
                        float a[2], bb[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float t1 = bf16_round(qkv_biased(p, col0 + c + e, acc[4 * j + 2 * h + e]));
                            const float t2 = bf16_round(qkv_biased(p, col0 + 64 + c + e, acc[4 * (j + 8) + 2 * h + e]));
                            rope_pair(t1, t2, csv[e], snv[e], a[e], bb[e]);
                        }
                        __nv_bfloat16* dst = gqa_qk_dst(p, row, col0 + c);
                        *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(a[0], a[1]);
                        *reinterpret_cast<uint32_t*>(dst + 64) = pack_bf16x2(bb[0], bb[1]);
                    }
                } else {
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int j = head * 16 + jj, col = col0 + 8 * jj + c0;
                        __nv_bfloat16* dst = gqa_vt_dst(p, col, b, pos);
                        dst[0] = __float2bfloat16_rn(qkv_biased(p, col, acc[4 * j + 2 * h]));
                        dst[p.Lpad] = __float2bfloat16_rn(qkv_biased(p, col + 1, acc[4 * j + 2 * h + 1]));
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Split-K tail: finishing pass. The S units of a tail tile have published their fp32 partial accumulators in the
// workspace; unit `s` owns the tile rows [128*s/S, 128*(s+1)/S) and, with all kEpiThreads epilogue threads, sums the partials of
// those rows in split order 0..S-1 (fixed -> deterministic; every load of an item is in flight before the first add) and
// applies the ordinary fused epilogue. Work items are (row, 8-column group) - for the rotary / SwiGLU epilogues the
// group's partner columns (+64 / +128) are fetched with it - and consecutive threads take consecutive rows of one group.
// ------------------------------------------------------------------------------------------------------------------
static constexpr int kSkMaxSplits = 8;
static constexpr int kEpiThreads = 256;  // the two MMA warpgroups of gemm.cu run the finishing pass

template <int BN, int NV>
__device__ __forceinline__ void sk_sum(const float4* __restrict__ tile_ws, int S, int row, const int (&col4)[NV], float4 (&acc)[NV]) {
    constexpr int kSplitStride = (BN / 4) * 128;  // float4 per split
    constexpr int kBatch = 4;                     // splits whose loads are in flight together (register budget)
    static_assert(kSkMaxSplits % kBatch == 0, "batches");
#pragma unroll
    for (int b0 = 0; b0 < kSkMaxSplits; b0 += kBatch) {
        if (b0 < S) {
            float4 part[kBatch][NV];
#pragma unroll
            for (int j = 0; j < kBatch; ++j)
                if (b0 + j < S) {
#pragma unroll
                    for (int v = 0; v < NV; ++v) part[j][v] = __ldcg(tile_ws + (size_t)(b0 + j) * kSplitStride + col4[v] * 128 + row);
                }
#pragma unroll
            for (int j = 0; j < kBatch; ++j)
                if (b0 + j < S) {
#pragma unroll
                    for (int v = 0; v < NV; ++v) {
                        if (b0 + j == 0) {
                            acc[v] = part[0][v];
                        } else {
                            acc[v].x = __fadd_rn(acc[v].x, part[j][v].x);
                            acc[v].y = __fadd_rn(acc[v].y, part[j][v].y);
                            acc[v].z = __fadd_rn(acc[v].z, part[j][v].z);
                            acc[v].w = __fadd_rn(acc[v].w, part[j][v].w);
                        }
                    }
                }
        }
    }
}

// publish this thread's accumulator fragment into split slot `slot_ws` ([BN/4][128] float4, viewed as floats)
template <int BN>
__device__ __forceinline__ void sk_publish(float* __restrict__ slot_ws, const float (&acc)[BN / 2], int rit0, int c0) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = 8 * j + c0;
            *reinterpret_cast<float2*>(slot_ws + ((size_t)(col >> 2) * 128 + rit0 + 8 * h) * 4 + (col & 3)) =
                make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
}

// cos / sin of position `pos`, table columns c .. c + 7 (the rotary item's angles)
__device__ __forceinline__ void rope_cs_load(const GemmParams& p, int pos, int c, float4 (&cs)[2], float4 (&sn)[2]) {
    const float4* c4 = reinterpret_cast<const float4*>(p.cos_tab + (size_t)pos * 64 + c);
    const float4* s4 = reinterpret_cast<const float4*>(p.sin_tab + (size_t)pos * 64 + c);
    cs[0] = c4[0]; cs[1] = c4[1]; sn[0] = s4[0]; sn[1] = s4[1];
}

// Rotary item of the QKV epilogues: q / k columns tc .. tc + 7 (v) and their partners tc + 64 .. (w) of GEMM row `row`
// (sequence b, position pos), with that position's cos / sin already loaded; stores 2 x 8 bf16.
template <int EPI, int BN>
__device__ __forceinline__ void qkv_rope_item(const GemmParams& p, int row, int b, int pos, int n_blk, int tc, const float (&v)[8],
                                              const float (&w)[8], const float4 (&cs4)[2], const float4 (&sn4)[2]) {
    const int n0 = n_blk * BN;
    const float cs[8] = {cs4[0].x, cs4[0].y, cs4[0].z, cs4[0].w, cs4[1].x, cs4[1].y, cs4[1].z, cs4[1].w};
    const float sn[8] = {sn4[0].x, sn4[0].y, sn4[0].z, sn4[0].w, sn4[1].x, sn4[1].y, sn4[1].z, sn4[1].w};
    float o1[8], o2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) rope_pair(bf16_round(v[i]), bf16_round(w[i]), cs[i], sn[i], o1[i], o2[i]);
    __nv_bfloat16* dst;
    if constexpr (epi_is_gqa(EPI)) {
        dst = gqa_qk_dst(p, row, n0 + tc);
    } else {
        const int region = n0 / p.d_model;  // 0 = Q, 1 = K (d_model % 256 == 0 is checked on the host)
        const size_t drow = (region == 0 || !p.pos_map) ? (size_t)row : (size_t)b * p.L + pos;  // k rows go to their sequence position
        dst = (region == 0 ? p.q : p.k) + drow * p.d_model + (n0 - region * p.d_model) + (tc >> 7) * 128 + (tc & 63);
    }
    *reinterpret_cast<uint4*>(dst) =
        make_uint4(pack_bf16x2(o1[0], o1[1]), pack_bf16x2(o1[2], o1[3]), pack_bf16x2(o1[4], o1[5]), pack_bf16x2(o1[6], o1[7]));
    *reinterpret_cast<uint4*>(dst + 64) =
        make_uint4(pack_bf16x2(o2[0], o2[1]), pack_bf16x2(o2[2], o2[3]), pack_bf16x2(o2[4], o2[5]), pack_bf16x2(o2[6], o2[7]));
}

// One work item of the fused epilogue, shared by the split-K finishing pass (fp32 sums) and the staged epilogue of
// gemm_bf16_kernel (bf16 values from shared memory; every epilogue rounds the accumulator to bf16 first, so both give the
// same bits as gemm_epilogue_tile): output row `row` (< p.M), 8 consecutive tile columns from `tc`, values v. The rotary and
// SwiGLU epilogues also take the partner columns w (tc + 64: the other rotary half; tc + 128: the up projection); `rv` is
// the residual at (row, n_blk * BN + tc) for EPI_RESID, loaded by the caller so that it can batch the loads of its items.
// Plain / residual / F32 and V items store 8 columns, rotary items 2 x 8, SwiGLU items the 8 products.
template <int EPI, int BN>
__device__ __forceinline__ void epi_row8(const GemmParams& p, int row, int n_blk, int tc, const float (&v)[8], const float (&w)[8],
                                         uint4 rv) {
    const int n0 = n_blk * BN;
    if constexpr (EPI == EPI_PLAIN || EPI == EPI_RESID || EPI == EPI_F32) {
        const int col = n0 + tc;
        if (col >= p.N) return;
        if constexpr (EPI == EPI_F32) {
            float4* d = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.C) + (size_t)row * p.ldc + col);
            d[0] = make_float4(v[0], v[1], v[2], v[3]);
            if (col + 4 < p.N) d[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
            uint32_t o[4];
            if constexpr (EPI == EPI_RESID) {
                const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    o[i] = pack_bf16x2(__fadd_rn(bf16_lo(rr[i]), bf16_round(v[2 * i])), __fadd_rn(bf16_hi(rr[i]), bf16_round(v[2 * i + 1])));
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) o[i] = pack_bf16x2(v[2 * i], v[2 * i + 1]);
            }
            *reinterpret_cast<uint4*>(p.C + (size_t)row * p.ldc + col) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    } else if constexpr (EPI == EPI_SWIGLU) {
        const int col = n_blk * (BN / 2) + tc;
        if (col >= p.N / 2) return;
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float gg = bf16_round(v[i]), uu = bf16_round(w[i]);
            const float sl = bf16_round(__fdiv_rn(gg, __fadd_rn(1.0f, expf(-gg))));  // silu -> bf16
            o[i] = __fmul_rn(sl, uu);
        }
        *reinterpret_cast<uint4*>(p.C + (size_t)row * p.ldc + col) =
            make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
    } else if constexpr (EPI == EPI_QKVROPE || EPI == EPI_QKVROPE_PACKED) {
        const int region = n0 / p.d_model;  // 0 = Q, 1 = K, 2 = V (d_model % 256 == 0 is checked on the host)
        int b, pos;
        qkv_row_coords<EPI>(p, row, b, pos);
        if (region < 2) {
            float4 cs[2], sn[2];
            rope_cs_load(p, pos, tc & 63, cs, sn);  // tc = head * 128 + c, c < 64
            qkv_rope_item<EPI, BN>(p, row, b, pos, n_blk, tc, v, w, cs, sn);
        } else {
            // V is written transposed: vt[b][head][d][token] so that P·V runs with both operands K-major
            const int n = n0 - 2 * p.d_model + tc;
            const int head = n >> 7, d0 = n & 127;
            __nv_bfloat16* dst = p.vt + ((size_t)(b * p.n_heads + head) * 128 + d0) * p.Lpad + pos;
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[(size_t)i * p.Lpad] = __float2bfloat16_rn(v[i]);
        }
    } else if constexpr (epi_is_gqa(EPI)) {
        // v / w already hold acc + bias (the caller adds it before any rounding)
        int b, pos;
        qkv_row_coords<EPI>(p, row, b, pos);
        const int col = n0 + tc;
        if (col < p.d_model + p.n_kv_heads * 128) {
            float4 cs[2], sn[2];
            rope_cs_load(p, pos, tc & 63, cs, sn);
            qkv_rope_item<EPI, BN>(p, row, b, pos, n_blk, tc, v, w, cs, sn);
        } else {
            __nv_bfloat16* dst = gqa_vt_dst(p, col, b, pos);
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[(size_t)i * p.Lpad] = __float2bfloat16_rn(v[i]);
        }
    }
}

// EPI_QKVGQA*: number of leading 128-column halves of tile n_blk that are q / k (rotary); the rest are V
template <int BN>
__device__ __forceinline__ int gqa_rot_halves(const GemmParams& p, int n_blk) {
    const int lim = p.d_model + p.n_kv_heads * 128 - n_blk * BN;
    return lim <= 0 ? 0 : (lim >= BN ? BN / 128 : lim / 128);
}

template <int EPI, int BN>
__device__ __forceinline__ void sk_finish(const GemmParams& p, const float4* __restrict__ tile_ws, int S, int unit_s, int m_blk,
                                          int n_blk, int tid) {
    const int r0 = (128 * unit_s) / S, r1 = (128 * (unit_s + 1)) / S;
    const int nrows = r1 - r0;
    if constexpr (epi_is_gqa(EPI)) {
        // per 128-column half: the rotary halves carry 8 paired items per row, the V halves 16 single ones
        const int nrot = gqa_rot_halves<BN>(p, n_blk);
        const int G = 8 * nrot + 16 * (BN / 128 - nrot);
        for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
            const int g = idx / nrows, rit = r0 + idx - g * nrows;
            const int row = m_blk * 128 + rit;
            if (row >= p.M) continue;
            const bool rot = g < 8 * nrot;
            const int tc = rot ? (g >> 3) * 128 + 8 * (g & 7) : 128 * nrot + 8 * (g - 8 * nrot);
            const int col = n_blk * BN + tc;
            if (col >= p.N) continue;
            float v[8], w[8];
            const int col4[4] = {tc / 4, tc / 4 + 1, (tc + 64) / 4, (tc + 64) / 4 + 1};
            float4 a[4];
            if (rot) sk_sum<BN, 4>(tile_ws, S, rit, col4, a);
            else {
                const int c2[2] = {col4[0], col4[1]};
                float4 a2[2];
                sk_sum<BN, 2>(tile_ws, S, rit, c2, a2);
                a[0] = a2[0]; a[1] = a2[1]; a[2] = a[3] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                v[4 * i] = a[i].x; v[4 * i + 1] = a[i].y; v[4 * i + 2] = a[i].z; v[4 * i + 3] = a[i].w;
                w[4 * i] = a[2 + i].x; w[4 * i + 1] = a[2 + i].y; w[4 * i + 2] = a[2 + i].z; w[4 * i + 3] = a[2 + i].w;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                v[i] = qkv_biased(p, col + i, v[i]);
                if (rot) w[i] = qkv_biased(p, col + 64 + i, w[i]);
            }
            epi_row8<EPI, BN>(p, row, n_blk, tc, v, w, make_uint4(0, 0, 0, 0));
        }
        return;
    }
    // items per tile row: 8-column groups; the rotary (q / k) and SwiGLU items carry their partner columns
    const bool pair = EPI == EPI_SWIGLU || ((EPI == EPI_QKVROPE || EPI == EPI_QKVROPE_PACKED) && n_blk * BN < 2 * p.d_model);
    const int G = pair ? 16 : BN / 8;
    for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
        const int g = idx / nrows, rit = r0 + idx - g * nrows;
        const int row = m_blk * 128 + rit;
        if (row >= p.M) continue;
        // tile column of the item and of its partner: SwiGLU g -> 8g, +128; rotary g = (head, gg) -> 128 head + 8 gg, +64
        const int tc = EPI == EPI_SWIGLU ? 8 * g : (pair ? (g >> 3) * 128 + 8 * (g & 7) : 8 * g);
        const int tw = EPI == EPI_SWIGLU ? tc + 128 : tc + 64;
        float v[8], w[8];
        if (pair) {
            const int col4[4] = {tc / 4, tc / 4 + 1, tw / 4, tw / 4 + 1};
            float4 a[4];
            sk_sum<BN, 4>(tile_ws, S, rit, col4, a);
            const float4 av[4] = {a[0], a[1], a[2], a[3]};
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                v[4 * i] = av[i].x; v[4 * i + 1] = av[i].y; v[4 * i + 2] = av[i].z; v[4 * i + 3] = av[i].w;
                w[4 * i] = av[2 + i].x; w[4 * i + 1] = av[2 + i].y; w[4 * i + 2] = av[2 + i].z; w[4 * i + 3] = av[2 + i].w;
            }
        } else {
            if (n_blk * BN + tc >= p.N) continue;
            const int col4[2] = {tc / 4, tc / 4 + 1};
            float4 a[2];
            sk_sum<BN, 2>(tile_ws, S, rit, col4, a);
#pragma unroll
            for (int i = 0; i < 2; ++i) { v[4 * i] = a[i].x; v[4 * i + 1] = a[i].y; v[4 * i + 2] = a[i].z; v[4 * i + 3] = a[i].w; }
#pragma unroll
            for (int i = 0; i < 8; ++i) w[i] = 0.f;
        }
        uint4 rv = make_uint4(0, 0, 0, 0);
        if constexpr (EPI == EPI_RESID) rv = *reinterpret_cast<const uint4*>(p.resid + (size_t)row * p.ldr + n_blk * BN + tc);
        epi_row8<EPI, BN>(p, row, n_blk, tc, v, w, rv);
    }
}

}  // namespace mmdp
