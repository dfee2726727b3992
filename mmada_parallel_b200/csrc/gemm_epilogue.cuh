// Fused epilogues of the bf16 GEMM kernel (gemm.cu). One call handles one thread's wgmma fragment of a 128 x BN
// accumulator tile held in registers.
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
};

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
            // tile columns [0,128) = gate rows of W1, [128,256) = up rows of W3 (weights packed interleaved)
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = n_blk * 128 + 8 * j + c0;
                if (col >= p.N / 2) continue;
                float o[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float gg = bf16_round(acc[4 * j + 2 * h + e]);
                    const float uu = bf16_round(acc[4 * (j + 16) + 2 * h + e]);
                    const float s = bf16_round(__fdiv_rn(gg, __fadd_rn(1.0f, expf(-gg))));  // silu -> bf16
                    o[e] = __fmul_rn(s, uu);
                }
                *reinterpret_cast<uint32_t*>(p.C + (size_t)row * p.ldc + col) = pack_bf16x2(o[0], o[1]);
            }
        } else if constexpr (EPI == EPI_QKVROPE) {
            const int region = n0 / p.d_model;  // 0 = Q, 1 = K, 2 = V (d_model % 256 == 0 is checked on the host)
            int b, pos;
            if (p.pos_map) {
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

template <int EPI, int BN>
__device__ __forceinline__ void sk_finish(const GemmParams& p, const float4* __restrict__ tile_ws, int S, int unit_s, int m_blk,
                                          int n_blk, int tid) {
    const int r0 = (128 * unit_s) / S, r1 = (128 * (unit_s + 1)) / S;
    const int nrows = r1 - r0;
    const int n0 = n_blk * BN;
    if constexpr (EPI == EPI_PLAIN || EPI == EPI_RESID || EPI == EPI_F32) {
        constexpr int G = BN / 8;
        for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
            const int g = idx / nrows, rit = r0 + idx - g * nrows;
            const int row = m_blk * 128 + rit, col = n0 + 8 * g;
            if (row >= p.M || col >= p.N) continue;
            const int col4[2] = {2 * g, 2 * g + 1};
            float4 a[2];
            sk_sum<BN, 2>(tile_ws, S, rit, col4, a);
            if constexpr (EPI == EPI_F32) {
                float4* d = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.C) + (size_t)row * p.ldc + col);
                d[0] = a[0];
                if (col + 4 < p.N) d[1] = a[1];
            } else {
                const float f[8] = {a[0].x, a[0].y, a[0].z, a[0].w, a[1].x, a[1].y, a[1].z, a[1].w};
                uint32_t o[4];
                if constexpr (EPI == EPI_RESID) {
                    const uint4 rv = *reinterpret_cast<const uint4*>(p.resid + (size_t)row * p.ldr + col);
                    const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        o[i] = pack_bf16x2(__fadd_rn(bf16_lo(rr[i]), bf16_round(f[2 * i])), __fadd_rn(bf16_hi(rr[i]), bf16_round(f[2 * i + 1])));
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) o[i] = pack_bf16x2(f[2 * i], f[2 * i + 1]);
                }
                *reinterpret_cast<uint4*>(p.C + (size_t)row * p.ldc + col) = make_uint4(o[0], o[1], o[2], o[3]);
            }
        }
    } else if constexpr (EPI == EPI_SWIGLU) {
        constexpr int G = 16;  // 128 output columns per tile
        for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
            const int g = idx / nrows, rit = r0 + idx - g * nrows;
            const int row = m_blk * 128 + rit, col = n_blk * 128 + 8 * g;
            if (row >= p.M || col >= p.N / 2) continue;
            const int col4[4] = {2 * g, 2 * g + 1, 32 + 2 * g, 32 + 2 * g + 1};
            float4 a[4];
            sk_sum<BN, 4>(tile_ws, S, rit, col4, a);
            const float gt[8] = {a[0].x, a[0].y, a[0].z, a[0].w, a[1].x, a[1].y, a[1].z, a[1].w};
            const float up[8] = {a[2].x, a[2].y, a[2].z, a[2].w, a[3].x, a[3].y, a[3].z, a[3].w};
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float gg = bf16_round(gt[i]), uu = bf16_round(up[i]);
                const float sl = bf16_round(__fdiv_rn(gg, __fadd_rn(1.0f, expf(-gg))));  // silu -> bf16
                o[i] = __fmul_rn(sl, uu);
            }
            *reinterpret_cast<uint4*>(p.C + (size_t)row * p.ldc + col) =
                make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
        }
    } else if constexpr (EPI == EPI_QKVROPE) {
        const int region = n0 / p.d_model;  // 0 = Q, 1 = K, 2 = V
        if (region < 2) {
            constexpr int G = 16;  // 2 heads x 8 column groups of the first half
            __nv_bfloat16* base = (region == 0 ? p.q : p.k) + (n0 - region * p.d_model);
            for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
                const int g = idx / nrows, rit = r0 + idx - g * nrows;
                const int row = m_blk * 128 + rit;
                if (row >= p.M) continue;
                const int head = g >> 3, gg = g & 7;
                const int col4[4] = {head * 32 + 2 * gg, head * 32 + 2 * gg + 1, head * 32 + 16 + 2 * gg, head * 32 + 16 + 2 * gg + 1};
                float4 a[4];
                sk_sum<BN, 4>(tile_ws, S, rit, col4, a);
                const int pos = (row + p.row0) % p.L;
                const float4* c4 = reinterpret_cast<const float4*>(p.cos_tab + (size_t)pos * 64 + 8 * gg);
                const float4* s4 = reinterpret_cast<const float4*>(p.sin_tab + (size_t)pos * 64 + 8 * gg);
                const float4 c0 = c4[0], c1 = c4[1], s0 = s4[0], s1 = s4[1];
                const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
                const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
                const float x1[8] = {a[0].x, a[0].y, a[0].z, a[0].w, a[1].x, a[1].y, a[1].z, a[1].w};
                const float x2[8] = {a[2].x, a[2].y, a[2].z, a[2].w, a[3].x, a[3].y, a[3].z, a[3].w};
                float o1[8], o2[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float t1 = bf16_round(x1[i]), t2 = bf16_round(x2[i]);
                    o1[i] = __fadd_rn(__fmul_rn(t1, cs[i]), __fmul_rn(-t2, sn[i]));
                    o2[i] = __fadd_rn(__fmul_rn(t2, cs[i]), __fmul_rn(t1, sn[i]));
                }
                __nv_bfloat16* dst = base + (size_t)row * p.d_model + head * 128 + 8 * gg;
                *reinterpret_cast<uint4*>(dst) =
                    make_uint4(pack_bf16x2(o1[0], o1[1]), pack_bf16x2(o1[2], o1[3]), pack_bf16x2(o1[4], o1[5]), pack_bf16x2(o1[6], o1[7]));
                *reinterpret_cast<uint4*>(dst + 64) =
                    make_uint4(pack_bf16x2(o2[0], o2[1]), pack_bf16x2(o2[2], o2[3]), pack_bf16x2(o2[4], o2[5]), pack_bf16x2(o2[6], o2[7]));
            }
        } else {
            constexpr int G = BN / 8;
            for (int idx = tid; idx < nrows * G; idx += kEpiThreads) {
                const int g = idx / nrows, rit = r0 + idx - g * nrows;
                const int row = m_blk * 128 + rit;
                if (row >= p.M) continue;
                const int col4[2] = {2 * g, 2 * g + 1};
                float4 a[2];
                sk_sum<BN, 2>(tile_ws, S, rit, col4, a);
                const int b = (row + p.row0) / p.L, pos = (row + p.row0) - b * p.L;
                const int n = n0 - 2 * p.d_model + 8 * g;
                const int head = n >> 7, d0 = n & 127;
                __nv_bfloat16* dst = p.vt + ((size_t)(b * p.n_heads + head) * 128 + d0) * p.Lpad + pos;
                const float f[8] = {a[0].x, a[0].y, a[0].z, a[0].w, a[1].x, a[1].y, a[1].z, a[1].w};
#pragma unroll
                for (int i = 0; i < 8; ++i) dst[(size_t)i * p.Lpad] = __float2bfloat16_rn(f[i]);
            }
        }
    }
}

}  // namespace mmdp
