// Attention forward (sm_90a): softmax(Q K^T / sqrt(128)) V for head_dim 128, no mask, whole-sequence KV.
//   * one CTA = one 128-row query tile of one (batch row, head); 384 threads: warpgroup 0 is the TMA producer (one elected
//     thread), warpgroups 1 and 2 each own 64 query rows;
//   * KV blocks of 128 keys, K and V^T double-buffered in shared memory (Q 32 KB + 2 x (32 + 32) KB = 160 KB, one CTA per SM);
//   * S = Q K^T with wgmma m64n128k16 (both operands from shared memory), the online softmax on the register fragment
//     (a query row is spread over the four lanes of a quad), P rounded to bf16 in registers and fed straight back as the A
//     operand of O += P V (wgmma with A from registers, B = V^T from shared memory); O stays in registers for the whole loop;
//   * the tiles of a partial last wave are cut along the keys and merged by attention_combine_kernel (see attention_fwd);
//   * attention_packed_kernel runs the same body over a packed variable-length batch: work items enumerate
//     (sequence, head, query tile), each sequence attends to its own keys only (attention_packed_fwd);
//   * grouped-query attention (kGqa): query head h reads kv head h / kv_group of k [rows, 128 Hkv] and V^T [B][Hkv][128][Lpad];
//     separate kernels, so that the multi-head ones keep their code;
//   * attention_packed_window_kernel (kWin): a packed batch where sequence s queries only its rows [lo_s, hi_s) (against all of
//     its keys) and writes them to a compact output, the windows of all sequences end to end (last-block row windows).
#include "mmdp_internal.h"
#include "ptx.cuh"

#include <stdlib.h>

#include <map>
#include <mutex>
#include <utility>

namespace mmdp {

static constexpr int kAttnThreads = 384;
// Two generations share this kernel, selected with the "attn_version" option: 6 (default) = KV blocks of 128 keys;
// 7 = KV blocks of 64 keys (half the S / P registers and 96 KB of shared memory, twice the block hand-offs).
static constexpr int kQBytes = 128 * 128 * 2;    // 32 KB: two 64-column halves [128 query rows][64 d]
template <int BKV> struct AttnCfg {
    static constexpr int kKBytes = BKV * 128 * 2;  // two 64-column halves [BKV keys][64 d]
    static constexpr int kVBytes = 128 * BKV * 2;  // BKV / 64 halves [128 d][64 keys]
    static constexpr int kSmem = kQBytes + 2 * (kKBytes + kVBytes) + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Sequence table of a packed launch: sequence s has rows [start[s], start[s + 1]) of q / k / out and the V^T block s; its
// query tiles are work items [tile0[s], tile0[s + 1]) (before the split of the tail), ordered (head, query tile).
struct AttnSegs {
    int n;
    int start[kMaxSegs + 1];
    int tile0[kMaxSegs + 1];
};

// Row windows of a packed launch: sequence s's queries are its rows [q0[s], q0[s] + nq[s]); their outputs are rows
// [out0[s], out0[s] + nq[s]) of the compact output. segs.tile0 counts the windows' query tiles; keys stay whole sequences.
struct AttnWin {
    AttnSegs segs;
    int q0[kMaxSegs], nq[kMaxSegs], out0[kMaxSegs];
};

// One CTA's work item. kPacked = false: B sequences of L keys / Lq queries each, laid out batch row after batch row (the
// kernel parameters). kPacked = true: the sequences of `segs`, each with its own length (L = Lq = its length).
// kGqa: H / kv_group kv heads, query head h reads kv head h / kv_group. kWin (with kPacked, segs = &win->segs): the row windows
// of `win`.
template <int kBKV, bool kPacked, bool kGqa = false, bool kWin = false>
__device__ __forceinline__ void attention_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmVt,
                                               __nv_bfloat16* __restrict__ out, int H, int L, int d_model, float scale_log2,
                                               int n_full, int splits, float* __restrict__ part_ws, int Lq, const AttnSegs* segs,
                                               int kv_group = 1, const AttnWin* win = nullptr) {
    constexpr int kKBytes = AttnCfg<kBKV>::kKBytes, kVBytes = AttnCfg<kBKV>::kVBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + kQBytes;
    uint8_t* sV = sK + 2 * kKBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * kVBytes);
    uint64_t* q_full = bars + 0;
    uint64_t* k_full = bars + 1;   // [2]
    uint64_t* k_empty = bars + 3;  // [2]
    uint64_t* v_full = bars + 5;   // [2]
    uint64_t* v_empty = bars + 7;  // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    // work items: [0, n_full) whole (b, h, query tile) problems; then, for each of the remaining tiles (the partial last wave),
    // `splits` pieces that each cover a slice of the KV blocks and leave an un-normalised partial (O, m, l) in part_ws for
    // attention_combine_kernel. tile index = (b * H + h) * n_qt + qt.
    // L = number of keys per batch row; Lq = number of query rows per batch row (== L except in the token-cache forward)
    int n_qt = (Lq + 127) / 128;
    int n_kv_all = (L + kBKV - 1) / kBKV;
    int tile = blockIdx.x, piece = -1;
    if ((int)blockIdx.x >= n_full) {
        const int t = (int)blockIdx.x - n_full;
        tile = n_full + t / splits;
        piece = t - (t / splits) * splits;
    }
    // packed: the tile's sequence (a uniform scan of the small table), its first row and length; keys past its end are masked
    // through nvalid, query rows past it are not stored. kWin: the first query row q0 and the first output row o0 of its window
    int seg = 0, seg0 = 0, tl = tile, q0 = 0, o0 = 0;
    if constexpr (kPacked) {
        for (int i = 1; i < segs->n; ++i)
            if (tile >= segs->tile0[i]) seg = i;
        seg0 = segs->start[seg];
        L = Lq = segs->start[seg + 1] - seg0;
        o0 = seg0;
        if constexpr (kWin) {
            q0 = win->q0[seg];
            Lq = win->nq[seg];
            o0 = win->out0[seg];
        }
        n_qt = (Lq + 127) / 128;
        n_kv_all = (L + kBKV - 1) / kBKV;
        tl = tile - segs->tile0[seg];
    }
    const int qt = tl % n_qt, h = (tl / n_qt) % H, b = kPacked ? seg : tile / (n_qt * H);
    const int hk = kGqa ? h / kv_group : h, Hk = kGqa ? H / kv_group : H;  // kv head and kv head count
    int jb = 0, je = n_kv_all;
    if (piece >= 0) {
        const int per = (n_kv_all + splits - 1) / splits;
        jb = piece * per;
        je = (jb + per < n_kv_all) ? jb + per : n_kv_all;
    }
    const int n_kv = je - jb;  // >= 1: the host keeps every piece of every split tile non-empty

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmVt);
        mbar_init(q_full, 1);
        for (int s = 0; s < 2; ++s) {
            mbar_init(&k_full[s], 1);
            mbar_init(&k_empty[s], 8);  // one arrive per MMA warp
            mbar_init(&v_full[s], 1);
            mbar_init(&v_empty[s], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();  // the prologue above overlaps the tail of the QKV GEMM (programmatic dependent launch)
    pdl_wait();

    if (wg == 0) {
        // ===================== TMA producer: Q, then K(j) and V^T(j) =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one_sync()) {
            const int qrow0 = (kPacked ? seg0 + q0 : b * Lq) + qt * 128;
            mbar_expect_tx(q_full, kQBytes);
            tma_load_2d(sQ, &tmQ, q_full, h * 128, qrow0);
            tma_load_2d(sQ + kQBytes / 2, &tmQ, q_full, h * 128 + 64, qrow0);
            for (int j = 0; j < n_kv; ++j) {
                const int st = j & 1;
                const uint32_t ph = (j >> 1) & 1;
                const int kv0 = (jb + j) * kBKV;
                mbar_wait(&k_empty[st], ph ^ 1);
                mbar_expect_tx(&k_full[st], kKBytes);
                tma_load_2d(sK + st * kKBytes, &tmK, &k_full[st], hk * 128, (kPacked ? seg0 : b * L) + kv0);
                tma_load_2d(sK + st * kKBytes + kKBytes / 2, &tmK, &k_full[st], hk * 128 + 64, (kPacked ? seg0 : b * L) + kv0);
                mbar_wait(&v_empty[st], ph ^ 1);
                mbar_expect_tx(&v_full[st], kVBytes);
                tma_load_2d(sV + st * kVBytes, &tmVt, &v_full[st], kv0, (b * Hk + hk) * 128);
                if (kBKV == 128) tma_load_2d(sV + st * kVBytes + kVBytes / 2, &tmVt, &v_full[st], kv0 + 64, (b * Hk + hk) * 128);
            }
        }
        __syncwarp();
        return;
    }

    // ===================== MMA + softmax (warpgroups 1, 2) =====================
    setmaxnreg_inc<232>();
    const int half = wg - 1;
    // fragment rows: r0 (h = 0) and r0 + 8 (h = 1) of the CTA's 128-row query tile; columns 8 jj + c0 + e
    const int r0 = half * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    const uint32_t aQ = smem_u32(sQ) + half * (64 * 128);
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);
    for (int j = 0; j < n_kv; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        const int nvalid = L - (jb + j) * kBKV;
        // S = Q K(j)^T (64 x 128 per warpgroup), K = head_dim 128: two 64-column halves of Q and K
        float sacc[kBKV / 2];
        const uint32_t aK = smem_u32(sK + st * kKBytes);
        mbar_wait(&k_full[st], ph);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
        {
            const uint64_t qd = smem_desc_kmajor_sw128(aQ + (kk >> 2) * (kQBytes / 2)) + (kk & 3) * 2;
            const uint64_t kd = smem_desc_kmajor_sw128(aK + (kk >> 2) * (kKBytes / 2)) + (kk & 3) * 2;
            if constexpr (kBKV == 128) wgmma_bf16_ss_n128(sacc, qd, kd, kk != 0);
            else wgmma_bf16_ss_n64(sacc, qd, kd, kk != 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(sacc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[st]);
        if (nvalid < kBKV) {
#pragma unroll
            for (int jj = 0; jj < kBKV / 8; ++jj)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (8 * jj + c0 + e >= nvalid) { sacc[4 * jj + e] = -INFINITY; sacc[4 * jj + 2 + e] = -INFINITY; }
        }
        // online softmax: running max per row (quad reduction), P = 2^((s - m) c), row sums in fp32 of the unrounded P
        float alpha[2], mneg[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float mx = sacc[2 * hh];
#pragma unroll
            for (int jj = 0; jj < kBKV / 8; ++jj) mx = fmaxf(mx, fmaxf(sacc[4 * jj + 2 * hh], sacc[4 * jj + 2 * hh + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[hh], mx);
            alpha[hh] = ex2_approx((m_run[hh] - m_new) * scale_log2);  // 0 on the first block (m_run = -inf)
            m_run[hh] = m_new;
            mneg[hh] = -m_new * scale_log2;
        }
        // P as the A fragments of the PV wgmma: k-step kk covers keys [16 kk, 16 kk + 16) = fragment columns jj = 2 kk, 2 kk + 1
        uint32_t pa[kBKV / 4];
        float rsum[2] = {0.f, 0.f};
#pragma unroll
        for (int jj = 0; jj < kBKV / 8; ++jj)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const float p0 = ex2_approx(fmaf(sacc[4 * jj + 2 * hh], scale_log2, mneg[hh]));
                const float p1 = ex2_approx(fmaf(sacc[4 * jj + 2 * hh + 1], scale_log2, mneg[hh]));
                rsum[hh] += p0 + p1;
                pa[2 * jj + hh] = pack_bf16x2(p0, p1);
            }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) l_run[hh] = fmaf(l_run[hh], alpha[hh], rsum[hh]);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
            o[4 * jj] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
            o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
        }
        // O += P V(j): B = V^T tile, [128 d][64 keys] per half, K-major
        const uint32_t aV = smem_u32(sV + st * kVBytes);
        mbar_wait(&v_full[st], ph);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBKV / 16; ++kk) {
            const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
            wgmma_bf16_rs_n128(o, a, smem_desc_kmajor_sw128(aV + (kk >> 2) * (kVBytes / 2)) + (kk & 3) * 2, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 1);
        l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh, qrow = qt * 128 + r;
        if (qrow >= Lq) continue;
        if (piece >= 0) {
            // partial result of this KV slice: O un-normalised (scaled by 2^(-m c)), m, l - merged by the combine kernel
            float* slot = part_ws + (size_t)((tile - n_full) * splits + piece) * (128 * 128 + 256);
            if ((lane & 3) == 0) {
                slot[128 * 128 + r] = m_run[hh];
                slot[128 * 128 + 128 + r] = l_run[hh];
            }
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
                *reinterpret_cast<float2*>(slot + (size_t)r * 128 + 8 * jj + c0) = make_float2(o[4 * jj + 2 * hh], o[4 * jj + 2 * hh + 1]);
        } else {
            const float inv_l = 1.0f / l_run[hh];
            __nv_bfloat16* orow = out + (size_t)((kPacked ? o0 : b * Lq) + qrow) * d_model + h * 128;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
                *reinterpret_cast<uint32_t*>(orow + 8 * jj + c0) = pack_bf16x2(o[4 * jj + 2 * hh] * inv_l, o[4 * jj + 2 * hh + 1] * inv_l);
        }
    }
}

template <int kBKV>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmVt, __nv_bfloat16* __restrict__ out, int H, int L, int d_model,
                 float scale_log2, int n_full, int splits, float* __restrict__ part_ws, int Lq) {
    attention_body<kBKV, false>(tmQ, tmK, tmVt, out, H, L, d_model, scale_log2, n_full, splits, part_ws, Lq, nullptr);
}

template <int kBKV>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_packed_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmVt, __nv_bfloat16* __restrict__ out, int H, int d_model,
                        float scale_log2, int n_full, int splits, float* __restrict__ part_ws, const __grid_constant__ AttnSegs segs) {
    attention_body<kBKV, true>(tmQ, tmK, tmVt, out, H, 0, d_model, scale_log2, n_full, splits, part_ws, 0, &segs);
}

template <int kBKV>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_gqa_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmVt, __nv_bfloat16* __restrict__ out, int H, int L, int d_model,
                     float scale_log2, int n_full, int splits, float* __restrict__ part_ws, int Lq, int kv_group) {
    attention_body<kBKV, false, true>(tmQ, tmK, tmVt, out, H, L, d_model, scale_log2, n_full, splits, part_ws, Lq, nullptr, kv_group);
}

template <int kBKV>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_packed_gqa_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                            const __grid_constant__ CUtensorMap tmVt, __nv_bfloat16* __restrict__ out, int H, int d_model,
                            float scale_log2, int n_full, int splits, float* __restrict__ part_ws, const __grid_constant__ AttnSegs segs,
                            int kv_group) {
    attention_body<kBKV, true, true>(tmQ, tmK, tmVt, out, H, 0, d_model, scale_log2, n_full, splits, part_ws, 0, &segs, kv_group);
}

// multi-head (kGqa = false, kv_group unused) and grouped-query instantiations of the windowed packed launch
template <int kBKV, bool kGqa>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_packed_window_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                               const __grid_constant__ CUtensorMap tmVt, __nv_bfloat16* __restrict__ out, int H, int d_model,
                               float scale_log2, int n_full, int splits, float* __restrict__ part_ws, const __grid_constant__ AttnWin win,
                               int kv_group) {
    attention_body<kBKV, true, kGqa, true>(tmQ, tmK, tmVt, out, H, 0, d_model, scale_log2, n_full, splits, part_ws, 0, &win.segs,
                                           kv_group, &win);
}

// Merges the `splits` KV-slice partials of one split tile: out = (sum_i w_i O_i) / (sum_i w_i l_i), w_i = 2^((m_i - m) c).
// One CTA per (split tile, query row), thread = output column.
template <bool kPacked, bool kWin = false>
__device__ __forceinline__ void attention_combine_body(const float* __restrict__ part_ws, __nv_bfloat16* __restrict__ out, int H,
                                                       int Lq, int d_model, float scale_log2, int n_full, int splits,
                                                       const AttnSegs* segs, const AttnWin* win = nullptr) {
    int n_qt = (Lq + 127) / 128;
    const int st = blockIdx.x, r = blockIdx.y, c = threadIdx.x;
    pdl_launch_dependents();
    pdl_wait();
    const int tile = n_full + st;
    int seg = 0, seg0 = 0, tl = tile;
    if constexpr (kPacked) {
        for (int i = 1; i < segs->n; ++i)
            if (tile >= segs->tile0[i]) seg = i;
        seg0 = segs->start[seg];
        Lq = segs->start[seg + 1] - seg0;
        if constexpr (kWin) {
            seg0 = win->out0[seg];  // output rows of the window
            Lq = win->nq[seg];
        }
        n_qt = (Lq + 127) / 128;
        tl = tile - segs->tile0[seg];
    }
    const int qt = tl % n_qt, h = (tl / n_qt) % H, b = kPacked ? seg : tile / (n_qt * H);
    const int qrow = qt * 128 + r;
    if (qrow >= Lq) return;
    const float* base = part_ws + (size_t)st * splits * (128 * 128 + 256);
    float m = -INFINITY;
    for (int i = 0; i < splits; ++i) m = fmaxf(m, base[(size_t)i * (128 * 128 + 256) + 128 * 128 + r]);
    float o = 0.f, l = 0.f;
    for (int i = 0; i < splits; ++i) {
        const float* slot = base + (size_t)i * (128 * 128 + 256);
        const float w = exp2f((slot[128 * 128 + r] - m) * scale_log2);
        o = fmaf(w, slot[(size_t)r * 128 + c], o);
        l = fmaf(w, slot[128 * 128 + 128 + r], l);
    }
    out[(size_t)((kPacked ? seg0 : b * Lq) + qrow) * d_model + h * 128 + c] = __float2bfloat16_rn(o / l);
}

__global__ void __launch_bounds__(128)
attention_combine_kernel(const float* __restrict__ part_ws, __nv_bfloat16* __restrict__ out, int H, int Lq, int d_model,
                         float scale_log2, int n_full, int splits) {
    attention_combine_body<false>(part_ws, out, H, Lq, d_model, scale_log2, n_full, splits, nullptr);
}

__global__ void __launch_bounds__(128)
attention_packed_combine_kernel(const float* __restrict__ part_ws, __nv_bfloat16* __restrict__ out, int H, int d_model,
                                float scale_log2, int n_full, int splits, const __grid_constant__ AttnSegs segs) {
    attention_combine_body<true>(part_ws, out, H, 0, d_model, scale_log2, n_full, splits, &segs);
}

__global__ void __launch_bounds__(128)
attention_packed_window_combine_kernel(const float* __restrict__ part_ws, __nv_bfloat16* __restrict__ out, int H, int d_model,
                                       float scale_log2, int n_full, int splits, const __grid_constant__ AttnWin win) {
    attention_combine_body<true, true>(part_ws, out, H, 0, d_model, scale_log2, n_full, splits, &win.segs, &win);
}

// KV-slice partials of the split tail: one buffer per (device, stream), grown on demand
static std::map<std::pair<int, cudaStream_t>, std::pair<float*, size_t>> g_attn_ws;
static std::mutex g_attn_ws_mu;
static int attn_part_workspace(cudaStream_t stream, size_t need, float** out) {
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_attn_ws_mu);
    auto& e = g_attn_ws[std::make_pair(dev, stream)];
    if (need > e.second) {
        if (e.first) MMDP_CUDA(cudaFree(e.first));  // synchronises with the launches that still read it
        e.first = nullptr; e.second = 0;
        MMDP_CUDA(cudaMalloc(&e.first, need));
        e.second = need;
    }
    *out = e.first;
    return 0;
}

// Partial last wave: tiles % SMs leftover tiles would run alone at the end. Split their KV range over the idle SMs and merge
// the partials (attention_combine_kernel). kvb_of(t) = number of KV blocks of work item t; every piece of every split tile
// must be non-empty for its own KV length.
template <class KvbOf>
static void plan_split_tail(int tiles, KvbOf kvb_of, int& n_full, int& n_split, int& splits) {
    const int split_tail = opt(OPT_ATTN_SPLIT_TAIL), slots = num_sms();
    n_full = tiles; n_split = 0; splits = 1;
    auto fit_splits = [&](int want, int first) {
        int sp = want > 8 ? 8 : want;
        for (int t = first; t < tiles; ++t)
            if (sp > kvb_of(t) / 2) sp = kvb_of(t) / 2;
        // no empty piece: piece i covers KV blocks [i * per, (i + 1) * per) with per = ceil(n_kvb / splits)
        auto empty_piece = [&](int s) {
            for (int t = first; t < tiles; ++t) {
                const int n_kvb = kvb_of(t);
                if ((s - 1) * ((n_kvb + s - 1) / s) >= n_kvb) return true;
            }
            return false;
        };
        while (sp >= 2 && empty_piece(sp)) --sp;
        return sp;
    };
    if (split_tail && tiles > slots && (tiles % slots) > 0 && (tiles % slots) * 4 <= slots) {
        n_split = tiles % slots;
        splits = fit_splits(slots / n_split, tiles - n_split);
        if (splits >= 2) n_full = tiles - n_split; else { n_split = 0; splits = 1; }
    } else if (split_tail && tiles * 2 <= slots) {
        // fewer tiles than half the SMs (a tensor-parallel rank with 4 of the 32 heads): split EVERY tile's KV range so
        // that the whole machine works on the launch
        splits = fit_splits(slots / tiles, 0);
        if (splits >= 2) { n_split = tiles; n_full = 0; } else splits = 1;
    }
}

template <class Kernel>
static int attn_smem_attr(Kernel kernel, int smem, unsigned long long& attr_set) {  // attr_set: bit per device
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    if (!(attr_set >> (dev & 63) & 1ull)) {
        MMDP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_set |= 1ull << (dev & 63);
    }
    return 0;
}

template <int kBKV>
static int attention_launch(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out, int B, int H,
                            int L, int Lpad, float scale, cudaStream_t stream, int Lq, int Hkv) {
    constexpr int kAttnSmem = AttnCfg<kBKV>::kSmem;
    if (B <= 0 || H <= 0 || L <= 0) return set_error("attention: empty problem");
    if (Lq <= 0) Lq = L;
    if (Hkv <= 0) Hkv = H;
    if (Hkv > H || H % Hkv) return set_error("attention: n_kv_heads=%d must divide n_heads=%d", Hkv, H);
    if (Lpad < L || (Lpad % 8)) return set_error("attention: Lpad must be >= L and a multiple of 8");
    const int d_model = H * 128, d_kv = Hkv * 128;
    CUtensorMap tmQ, tmK, tmVt;
    if (make_tmap_2d_bf16(&tmQ, q, (uint64_t)B * Lq, (uint64_t)d_model, (uint64_t)d_model, 128, 64)) return -1;
    if (make_tmap_2d_bf16(&tmK, k, (uint64_t)B * L, (uint64_t)d_kv, (uint64_t)d_kv, kBKV, 64)) return -1;
    if (make_tmap_2d_bf16(&tmVt, vt, (uint64_t)B * Hkv * 128, (uint64_t)Lpad, (uint64_t)Lpad, 128, 64)) return -1;
    const int n_qt = (Lq + 127) / 128, n_kvb = (L + kBKV - 1) / kBKV;
    const int tiles = n_qt * H * B;
    int n_full, n_split, splits;
    plan_split_tail(tiles, [&](int) { return n_kvb; }, n_full, n_split, splits);
    float* part_ws = nullptr;
    if (n_split > 0 && attn_part_workspace(stream, (size_t)n_split * splits * (128 * 128 + 256) * sizeof(float), &part_ws)) return -1;
    const int grid = n_full + n_split * splits;
    const float scale_log2 = scale * 1.4426950408889634f;
    const bool pdl = pdl_mode() != 0;
    LaunchScope ls(LK_ATTN, 4.0 * B * H * (double)Lq * L * 128, stream);
    if (Hkv != H) {
        static unsigned long long attr_set_gqa = 0;
        if (attn_smem_attr(attention_gqa_kernel<kBKV>, kAttnSmem, attr_set_gqa)) return -1;
        MMDP_CUDA(launch_ex(attention_gqa_kernel<kBKV>, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, pdl, false, tmQ, tmK, tmVt, out,
                            H, L, d_model, scale_log2, n_full, splits, part_ws, Lq, H / Hkv));
    } else {
        static unsigned long long attr_set = 0;
        if (attn_smem_attr(attention_kernel<kBKV>, kAttnSmem, attr_set)) return -1;
        MMDP_CUDA(launch_ex(attention_kernel<kBKV>, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, pdl, false, tmQ, tmK, tmVt, out, H, L,
                            d_model, scale_log2, n_full, splits, part_ws, Lq));
    }
    if (n_split > 0)
        MMDP_CUDA(launch_ex(attention_combine_kernel, dim3(n_split, 128), dim3(128), 0, stream, pdl, false, (const float*)part_ws, out, H, Lq,
                            d_model, scale_log2, n_full, splits));
    return 0;
}

// win_lo / win_hi (host, both null or both set): sequence s queries its rows [win_lo[s], win_hi[s]) only, and `out` is compact
template <int kBKV>
static int attention_packed_launch(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out,
                                   const SegTable& segs, int H, int Lpad, float scale, cudaStream_t stream, int Hkv,
                                   const int* win_lo, const int* win_hi) {
    constexpr int kAttnSmem = AttnCfg<kBKV>::kSmem;
    if (segs.n <= 0 || segs.n > kMaxSegs || H <= 0) return set_error("attention_packed: %d sequences (1 to %d)", segs.n, kMaxSegs);
    if (Hkv <= 0) Hkv = H;
    if (Hkv > H || H % Hkv) return set_error("attention_packed: n_kv_heads=%d must divide n_heads=%d", Hkv, H);
    if (Lpad % 8) return set_error("attention_packed: Lpad must be a multiple of 8");
    if (!win_lo != !win_hi) return set_error("attention_packed: give both window bounds or neither");
    const bool windowed = win_lo != nullptr;
    AttnWin aw{};
    AttnSegs& as = aw.segs;
    as.n = segs.n;
    double work = 0;
    int Mq = 0;  // windowed: rows of the compact output
    for (int s = 0; s <= segs.n; ++s) {
        as.start[s] = segs.start[s];
        if (s == segs.n) break;
        const int len = segs.start[s + 1] - segs.start[s];
        if (len <= 0 || len > Lpad) return set_error("attention_packed: sequence %d has length %d (Lpad %d)", s, len, Lpad);
        const int lo = windowed ? win_lo[s] : 0, hi = windowed ? win_hi[s] : len;
        if (lo < 0 || lo >= hi || hi > len)
            return set_error("attention_packed: sequence %d of length %d has the row window [%d, %d)", s, len, lo, hi);
        aw.q0[s] = lo;
        aw.nq[s] = hi - lo;
        aw.out0[s] = Mq;
        Mq += hi - lo;
        as.tile0[s + 1] = as.tile0[s] + (hi - lo + 127) / 128 * H;
        work += 4.0 * H * (double)(hi - lo) * len * 128;
    }
    const int M = segs.start[segs.n], tiles = as.tile0[segs.n], d_model = H * 128, d_kv = Hkv * 128;
    CUtensorMap tmQ, tmK, tmVt;
    if (make_tmap_2d_bf16(&tmQ, q, (uint64_t)M, (uint64_t)d_model, (uint64_t)d_model, 128, 64)) return -1;
    if (make_tmap_2d_bf16(&tmK, k, (uint64_t)M, (uint64_t)d_kv, (uint64_t)d_kv, kBKV, 64)) return -1;
    if (make_tmap_2d_bf16(&tmVt, vt, (uint64_t)segs.n * Hkv * 128, (uint64_t)Lpad, (uint64_t)Lpad, 128, 64)) return -1;
    auto kvb_of = [&](int t) {
        int s = 0;
        while (s + 1 < segs.n && t >= as.tile0[s + 1]) ++s;
        return (segs.start[s + 1] - segs.start[s] + kBKV - 1) / kBKV;
    };
    int n_full, n_split, splits;
    plan_split_tail(tiles, kvb_of, n_full, n_split, splits);
    float* part_ws = nullptr;
    if (n_split > 0 && attn_part_workspace(stream, (size_t)n_split * splits * (128 * 128 + 256) * sizeof(float), &part_ws)) return -1;
    const int grid = n_full + n_split * splits;
    const float scale_log2 = scale * 1.4426950408889634f;
    const bool pdl = pdl_mode() != 0;
    LaunchScope ls(LK_ATTN, work, stream);
    if (windowed) {
        auto kernel = Hkv != H ? attention_packed_window_kernel<kBKV, true> : attention_packed_window_kernel<kBKV, false>;
        static unsigned long long attr_set_win[2] = {0, 0};
        if (attn_smem_attr(kernel, kAttnSmem, attr_set_win[Hkv != H])) return -1;
        MMDP_CUDA(launch_ex(kernel, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, pdl, false, tmQ, tmK, tmVt, out, H, d_model,
                            scale_log2, n_full, splits, part_ws, aw, H / Hkv));
        if (n_split > 0)
            MMDP_CUDA(launch_ex(attention_packed_window_combine_kernel, dim3(n_split, 128), dim3(128), 0, stream, pdl, false,
                                (const float*)part_ws, out, H, d_model, scale_log2, n_full, splits, aw));
        return 0;
    }
    if (Hkv != H) {
        static unsigned long long attr_set_gqa = 0;
        if (attn_smem_attr(attention_packed_gqa_kernel<kBKV>, kAttnSmem, attr_set_gqa)) return -1;
        MMDP_CUDA(launch_ex(attention_packed_gqa_kernel<kBKV>, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, pdl, false, tmQ, tmK, tmVt,
                            out, H, d_model, scale_log2, n_full, splits, part_ws, as, H / Hkv));
    } else {
        static unsigned long long attr_set = 0;
        if (attn_smem_attr(attention_packed_kernel<kBKV>, kAttnSmem, attr_set)) return -1;
        MMDP_CUDA(launch_ex(attention_packed_kernel<kBKV>, dim3(grid), dim3(kAttnThreads), kAttnSmem, stream, pdl, false, tmQ, tmK, tmVt, out,
                            H, d_model, scale_log2, n_full, splits, part_ws, as));
    }
    if (n_split > 0)
        MMDP_CUDA(launch_ex(attention_packed_combine_kernel, dim3(n_split, 128), dim3(128), 0, stream, pdl, false, (const float*)part_ws,
                            out, H, d_model, scale_log2, n_full, splits, as));
    return 0;
}

int attention_fwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out, int B, int H, int L,
                  int Lpad, float scale, cudaStream_t stream, int Lq, int Hkv) {
    const int version = opt(OPT_ATTN_VERSION);
    if (version == 7) return attention_launch<64>(q, k, vt, out, B, H, L, Lpad, scale, stream, Lq, Hkv);
    if (version != 6) return set_error("attention: unknown kernel generation %d (6 or 7)", version);
    return attention_launch<128>(q, k, vt, out, B, H, L, Lpad, scale, stream, Lq, Hkv);
}

int attention_packed_fwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* vt, __nv_bfloat16* out,
                         const SegTable& segs, int H, int Lpad, float scale, cudaStream_t stream, int Hkv, const int* win_lo,
                         const int* win_hi) {
    const int version = opt(OPT_ATTN_VERSION);
    if (version == 7) return attention_packed_launch<64>(q, k, vt, out, segs, H, Lpad, scale, stream, Hkv, win_lo, win_hi);
    if (version != 6) return set_error("attention: unknown kernel generation %d (6 or 7)", version);
    return attention_packed_launch<128>(q, k, vt, out, segs, H, Lpad, scale, stream, Hkv, win_lo, win_hi);
}

}  // namespace mmdp
