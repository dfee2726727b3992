// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = A[M,K] · W[N,K]^T  (fp32 accumulate in registers)
//
//   warpgroup 0    : TMA producer  (warp 0, one elected thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier
//                    complete_tx) and, in warps 1-3, the fused epilogue of the previous tile (staged epilogues)
//   warpgroups 1,2 : MMA (wgmma m64nBNk16, one 64-row half of the 128 x BN tile each). After the last k-block they write the
//                    tile as bf16 into a staging tile in shared memory and go straight on to the next tile's k-blocks; the
//                    epilogue warps apply the fused epilogue from there with 16-byte loads and stores. The fp32 partials
//                    (EPI_F32) and the split-K tail keep the epilogue on the register fragments.
//
// Every nn.Linear of the reference block (MMaDA-Parallel-A/model/modeling_llada.py:925-927, :744, :962, :968, :1402)
// maps to one launch of this kernel with a fused epilogue that reproduces the reference's bf16 rounding points:
//   EPI_PLAIN   : C = bf16(acc)                                            (LM head, :1402)
//   EPI_RESID   : C = bf16( bf16(acc) + resid )                            (attn_out + residual :744/:953; ff_out :968/:970)
//   EPI_QKVROPE : q,k = bf16( rope_fp32( bf16(acc) ) ), v^T = bf16(acc)    (q/k/v_proj :925-927 + RotaryEmbedding :402-435)
//   EPI_SWIGLU  : C = bf16( bf16(silu(bf16(g))) * bf16(u) )                (ff_proj/up_proj/act/mul :962-967)
//   EPI_QKVROPE_PACKED : EPI_QKVROPE over a packed variable-length batch (per-row sequence and position)
//   EPI_QKVGQA(_PACKED): the two above with grouped-query k / v and q,k,v = bf16(acc + bias)   (k/v_proj :872-884)
#include "gemm_epilogue.cuh"

#include <stdlib.h>

#include <map>
#include <mutex>
#include <utility>

namespace mmdp {

static constexpr int BM = 128, BK = 64;
static constexpr int kABytes = BM * BK * 2;  // 16 KB
static constexpr int kGemmThreads = 384;
static constexpr int kStagedEpiThreads = 96;  // warps 1-3 of the producer warpgroup run the staged epilogue
static constexpr int kStagedEpiRegs = 88;     // their register budget (setmaxnreg); the MMA warpgroups get the rest
// The N tile width is a template parameter: 256 (default; required by the QKV/SwiGLU epilogues) or 192. The K loop and
// therefore the fp32 accumulation order of every output element is identical for both, so results do not depend on
// the tile width; the host picks the width that minimises (waves x width) for the problem (wave quantisation on the SMs).
// kStaged: the tile leaves the MMA warps as bf16 through a staging tile in shared memory (128 rows of BN bf16, rows padded by
// 16 bytes) that the epilogue warps drain while the MMA warps run the next tile; the staging tile takes one ring stage.
template <int BN, bool kStaged> struct GemmCfg {
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (BN == 256 ? 4 : 5) - (kStaged ? 1 : 0);  // ring: 192 / 200 KB, staged 144 / 160 KB
    static constexpr int kStagingStride = BN * 2 + 16;
    static constexpr int kStagingBytes = kStaged ? BM * kStagingStride : 0;  // 66 / 50 KB
    static constexpr int kSmem = kStages * kStageBytes + kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(kSmem <= 227 * 1024, "an H100 block may use 227 KB of shared memory");
};
// every epilogue except the fp32 partials rounds the accumulator to bf16 first, so a bf16 staging tile is exact
template <int EPI> constexpr bool gemm_staged() { return EPI != EPI_F32; }

// MMA warps: this thread's fragment (gemm_epilogue_tile's mapping) into the staging tile as bf16 pairs. Banks: a warp's store
// covers 8 rows x 4 consecutive words; the row stride is BN / 2 + 4 words = 4 (mod 32), so the 32 words fall in 32 banks.
template <int BN>
__device__ __forceinline__ void stage_tile(uint8_t* stg, const float (&acc)[BN / 2], int rit0, int c0) {
    constexpr int kStride = GemmCfg<BN, true>::kStagingStride;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
            *reinterpret_cast<uint32_t*>(stg + (rit0 + 8 * h) * kStride + (8 * j + c0) * 2) = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
}

__device__ __forceinline__ void bf16x8_to_float(uint4 x, float (&f)[8]) {
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { f[2 * i] = bf16_lo(xs[i]); f[2 * i + 1] = bf16_hi(xs[i]); }
}

// V^T of a staged QKV tile: items are 8 rows x 8 columns. When the 8 rows are 8 consecutive positions of one sequence starting
// at a multiple of 8, the block is transposed in registers and each column (one d of V^T) is one 16-byte store; otherwise
// (a sequence boundary inside the 8 rows, a position map, rows past M) every row goes through epi_row8's element stores.
// Grouped-query tiles (EPI_QKVGQA*) pass cg0 = 16 x the tile's rotary halves: only the 8-column groups from cg0 on are V.
// `nthr` threads (etid < nthr) share the items. x is indexed with constants only, so it stays in registers. Eight consecutive
// threads take eight column groups of one 8-row group (their 16-byte staging reads fall in 32 distinct banks) and a warp
// covers four consecutive 8-row groups, so each column store of a warp writes 64 contiguous bytes (two whole sectors) into
// each of eight V^T rows instead of 16 bytes into each of 32.
template <int EPI, int BN>
__device__ __forceinline__ void staged_vt(const GemmParams& p, const uint8_t* stg, int m_blk, int n_blk, int etid, int nthr, int cg0 = 0) {
    constexpr int kStride = GemmCfg<BN, true>::kStagingStride;
    const int CG = BN / 8 - cg0;
    const bool aligned = (p.Lpad & 7) == 0 && (reinterpret_cast<uintptr_t>(p.vt) & 15) == 0;
    for (int idx = etid; idx < 16 * CG; idx += nthr) {
        const int rg = (idx >> 3) & 15, cg = cg0 + (idx & 7) + 8 * (idx >> 7);  // CG is 16 or 32
        const int r0 = m_blk * 128 + 8 * rg;
        if (r0 >= p.M) continue;
        uint4 x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = *reinterpret_cast<const uint4*>(stg + (8 * rg + i) * kStride + 16 * cg);
        int b0, pos0;
        qkv_row_coords<EPI>(p, r0, b0, pos0);
        bool vec = aligned && r0 + 7 < p.M && (pos0 & 7) == 0;
        if (epi_is_packed(EPI) || p.pos_map) {
            for (int i = 1; i < 8 && vec; ++i) {
                int b, pos;
                qkv_row_coords<EPI>(p, r0 + i, b, pos);
                vec = b == b0 && pos == pos0 + i;
            }
        } else {
            vec = vec && pos0 + 7 < p.L;  // rows r0 + i are positions pos0 + i of one sequence
        }
        if (vec) {
            const int n = n_blk * BN - (epi_is_gqa(EPI) ? p.d_model + p.n_kv_heads * 128 : 2 * p.d_model) + 8 * cg;
            const int head = n >> 7, d0 = n & 127;
            __nv_bfloat16* dst = p.vt + ((size_t)(b0 * (epi_is_gqa(EPI) ? p.n_kv_heads : p.n_heads) + head) * 128 + d0) * p.Lpad + pos0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                uint32_t o[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4 a = x[2 * k], b = x[2 * k + 1];
                    const uint32_t wa = (c >> 1) == 0 ? a.x : (c >> 1) == 1 ? a.y : (c >> 1) == 2 ? a.z : a.w;
                    const uint32_t wb = (c >> 1) == 0 ? b.x : (c >> 1) == 1 ? b.y : (c >> 1) == 2 ? b.z : b.w;
                    o[k] = __byte_perm(wa, wb, (c & 1) ? 0x7632 : 0x5410);  // column c of rows 2k (low half) and 2k + 1
                }
                *reinterpret_cast<uint4*>(dst + (size_t)c * p.Lpad) = make_uint4(o[0], o[1], o[2], o[3]);
            }
        } else {
            const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll 1
            for (int i = 0; i < 8; ++i) {
                if (r0 + i >= p.M) break;
                float v[8];
                bf16x8_to_float(x[0], v);
                epi_row8<EPI, BN>(p, r0 + i, n_blk, 8 * cg, v, v, zero);
#pragma unroll
                for (int j = 0; j < 7; ++j) x[j] = x[j + 1];  // row r0 + i + 1 moves to x[0]
            }
        }
    }
}

// The fused epilogue of one staged tile, shared by `nthr` threads (etid < nthr). Items are (row, 8-column group) as in the
// split-K finishing pass; consecutive threads take consecutive groups of a row, so a warp reads a row's 16-byte chunks (512
// contiguous bytes: no bank conflict) and its global loads and stores are whole 16-byte pieces of one or two rows. Plain and
// residual items run U at a time with all their loads issued before the first store (C may be the residual: the compiler
// cannot reorder them).
template <int EPI, int BN>
__device__ __forceinline__ void staged_epilogue(const GemmParams& p, const uint8_t* stg, int m_blk, int n_blk, int etid, int nthr) {
    constexpr int kStride = GemmCfg<BN, true>::kStagingStride;
    if constexpr (epi_is_qkv(EPI)) {
        int n_rot = BN / 128;  // rotary (q / k) halves of the tile; the rest is V
        if constexpr (epi_is_gqa(EPI)) n_rot = gqa_rot_halves<BN>(p, n_blk);
        else if (n_blk * BN >= 2 * p.d_model) n_rot = 0;
        if (n_rot < BN / 128) staged_vt<EPI, BN>(p, stg, m_blk, n_blk, etid, nthr, 16 * n_rot);
        if (n_rot == 0) return;
        // rotary items (row, 8-column group gg) span the tile's rotary halves: columns 128 h + 8 gg and their partners + 64
        // all take the cos / sin of (position, 8 gg), loaded once. Every load of an item (up to 4 staging chunks, the row's
        // position, 4 cos / sin chunks) is issued before its first store.
        for (int idx = etid; idx < BM * 8; idx += nthr) {
            const int rit = idx >> 3, gg = idx & 7;
            const int row = m_blk * BM + rit;
            if (row >= p.M) break;
            uint4 xv[BN / 128], xw[BN / 128];
#pragma unroll
            for (int h = 0; h < BN / 128; ++h) {
                if (h < n_rot) {
                    xv[h] = *reinterpret_cast<const uint4*>(stg + rit * kStride + (128 * h + 8 * gg) * 2);
                    xw[h] = *reinterpret_cast<const uint4*>(stg + rit * kStride + (128 * h + 8 * gg + 64) * 2);
                }
            }
            int sq, pos;
            qkv_row_coords<EPI>(p, row, sq, pos);
            float4 cs[2], sn[2];
            rope_cs_load(p, pos, 8 * gg, cs, sn);
#pragma unroll
            for (int h = 0; h < BN / 128; ++h) {
                if (h < n_rot) {
                    float v[8], w[8];
                    bf16x8_to_float(xv[h], v);
                    bf16x8_to_float(xw[h], w);
                    qkv_rope_item<EPI, BN>(p, row, sq, pos, n_blk, 128 * h + 8 * gg, v, w, cs, sn);
                }
            }
        }
    } else {
        constexpr bool kPair = EPI == EPI_SWIGLU;
        constexpr int G = kPair ? 16 : BN / 8;
        constexpr int kItems = BM * G;
        constexpr int U = kPair ? 1 : 4;
        for (int i0 = etid; i0 < kItems; i0 += U * nthr) {
            uint4 xv[U], xw[U], rv[U];
            int row[U], tc[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int idx = i0 + u * nthr;
                const int rit = idx / G, g = idx - rit * G;
                tc[u] = 8 * g;  // SwiGLU: gate columns 8g, up + 128
                row[u] = (idx < kItems && m_blk * BM + rit < p.M) ? m_blk * BM + rit : -1;
                rv[u] = make_uint4(0, 0, 0, 0);
                if (row[u] < 0) continue;
                xv[u] = *reinterpret_cast<const uint4*>(stg + rit * kStride + tc[u] * 2);
                if constexpr (kPair) xw[u] = *reinterpret_cast<const uint4*>(stg + rit * kStride + (tc[u] + 128) * 2);
                if constexpr (EPI == EPI_RESID) {
                    if (n_blk * BN + tc[u] < p.N) rv[u] = *reinterpret_cast<const uint4*>(p.resid + (size_t)row[u] * p.ldr + n_blk * BN + tc[u]);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (row[u] < 0) continue;
                float v[8], w[8];
                bf16x8_to_float(xv[u], v);
                if constexpr (kPair) bf16x8_to_float(xw[u], w);
                epi_row8<EPI, BN>(p, row[u], n_blk, tc[u], v, kPair ? w : v, rv[u]);
            }
        }
    }
}

template <int EPI, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    constexpr bool kStaged = gemm_staged<EPI>();
    constexpr int kStages = GemmCfg<BN, kStaged>::kStages;
    constexpr int kStageBytes = GemmCfg<BN, kStaged>::kStageBytes;
    static_assert(EPI == EPI_PLAIN || EPI == EPI_RESID || EPI == EPI_F32 || BN == 256, "fused QKV / SwiGLU epilogues need 256-wide tiles");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* staging = smem + kStages * kStageBytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + GemmCfg<BN, kStaged>::kStagingBytes);
    uint64_t* empty_bar = full_bar + kStages;
    // staged epilogue: "staged" completes when the MMA warps have written a tile into the staging tile, "drained" when the
    // epilogue warps have read it; the k-th full tile of this CTA completes phase k of each
    uint64_t* staged_bar = empty_bar + kStages;
    uint64_t* drained_bar = staged_bar + 1;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrive per MMA warp
        }
        if constexpr (kStaged) {
            mbar_init(staged_bar, 256);                 // every MMA thread, after its stores
            mbar_init(drained_bar, kStagedEpiThreads);  // every epilogue thread, after its loads
        }
        fence_barrier_init();
    }
    __syncthreads();
    // everything above overlaps the tail of the previous kernel in the stream (programmatic dependent launch)
    pdl_launch_dependents();
    pdl_wait();

    const int num_m = (p.M + BM - 1) / BM;
    const int num_n = (p.N + BN - 1) / BN;
    const int num_k = (p.K + BK - 1) / BK;
    const int num_tiles = num_m * num_n;
    // tiles [0, full_tiles) are computed whole (persistent loop); the remaining p.sk_tail tiles - a partial last wave -
    // are split along K: unit u = blockIdx.x handles tile full_tiles + u / splits, k-blocks [kb0, kb1)
    const int full_tiles = num_tiles - p.sk_tail;
    const bool has_unit = p.sk_tail > 0 && (int)blockIdx.x < p.sk_tail * p.sk_splits;
    const int unit_t = has_unit ? (int)blockIdx.x / p.sk_splits : 0;
    const int unit_s = has_unit ? (int)blockIdx.x - unit_t * p.sk_splits : 0;
    const int unit_tile = full_tiles + unit_t;
    const int unit_kb0 = unit_s * p.sk_kb_per;
    const int unit_kb1 = (unit_kb0 + p.sk_kb_per < num_k) ? unit_kb0 + p.sk_kb_per : num_k;

    if (wg == 0) {
        // ===================== TMA producer (warp 0) and staged epilogue (warps 1-3) =====================
        // staged: 88 / 208 / 208 registers per thread (64 512 of the 65 536 for 384 threads): the epilogue warps keep a
        // rotary item's loads (4 staging chunks, 4 cos / sin chunks) and V^T's 8 x 8 block in registers without spilling
        setmaxnreg_dec<kStaged ? kStagedEpiRegs : 40>();
        if constexpr (kStaged) {
            if (warp > 0) {
                const int etid = threadIdx.x - 32;
                uint32_t it = 0;
                for (int tile = blockIdx.x; tile < full_tiles; tile += gridDim.x, ++it) {  // the split-K unit never stages
                    int m_blk, n_blk;
                    gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
                    mbar_wait(staged_bar, it & 1);
                    const bool shared = !has_unit && tile + (int)gridDim.x >= full_tiles;  // the MMA warps join (below)
                    staged_epilogue<EPI, BN>(p, staging, m_blk, n_blk, etid, shared ? kStagedEpiThreads + 256 : kStagedEpiThreads);
                    mbar_arrive(drained_bar);
                }
            }
        }
        if (warp == 0 && elect_one_sync()) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < full_tiles + (has_unit ? 1 : 0) * gridDim.x; tile += gridDim.x) {
                const bool is_unit = tile >= full_tiles;
                const int tl = is_unit ? unit_tile : tile;
                int m_blk, n_blk;
                gemm_tile_coords(tl, num_m, num_n, p.group_m, m_blk, n_blk);
                const int kb_beg = is_unit ? unit_kb0 : 0, kb_end = is_unit ? unit_kb1 : num_k;
                // weight tiles are prefetched into L2 `l2pf` k-blocks ahead by every l2pf_mod-th m-tile's CTA (the CTAs that
                // share an n-tile run in lock-step, so one of them fetching ahead turns the others' DRAM misses into L2 hits)
                const bool pf = p.l2pf > 0 && ((m_blk + n_blk) % p.l2pf_mod) == 0;
                for (int kb = kb_beg; kb < kb_end; ++kb) {
                    if (pf && kb + p.l2pf < kb_end) tma_prefetch_l2_2d(&tmB, (kb + p.l2pf) * BK, n_blk * BN);
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], kStageBytes);
                    uint8_t* sa = smem + s * kStageBytes;
                    tma_load_2d(sa, &tmA, &full_bar[s], kb * BK, m_blk * BM);
                    tma_load_2d(sa + kABytes, &tmB, &full_bar[s], kb * BK, n_blk * BN);
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
                if (is_unit) break;
            }
        }
        __syncwarp();
    } else {
        // ===================== MMA + epilogue (warpgroups 1 and 2: tile rows [64 (wg-1), 64 wg)) =====================
        setmaxnreg_inc<kStaged ? (64512 - 128 * kStagedEpiRegs) / 256 : 232>();
        const int half = wg - 1;
        const int rit0 = half * 64 + (warp & 3) * 16 + (lane >> 2);  // tile row of acc[4j + 0..1]; acc[4j + 2..3] is 8 rows below
        const int c0 = 2 * (lane & 3);
        float acc[BN / 2];
        int s = 0;
        uint32_t ph = 0;
        uint32_t it = 0;  // full tiles staged so far
        int last_m = -1, last_n = 0;  // the last staged tile
        for (int tile = blockIdx.x; tile < full_tiles + (has_unit ? 1 : 0) * gridDim.x; tile += gridDim.x) {
            const bool is_unit = tile >= full_tiles;
            const int tl = is_unit ? unit_tile : tile;
            int m_blk, n_blk;
            gemm_tile_coords(tl, num_m, num_n, p.group_m, m_blk, n_blk);
            const int kb_beg = is_unit ? unit_kb0 : 0, kb_end = is_unit ? unit_kb1 : num_k;
            int prev_s = -1;
            for (int kb = kb_beg; kb < kb_end; ++kb) {
                mbar_wait(&full_bar[s], ph);
                const uint32_t sa = smem_u32(smem + s * kStageBytes);
                const uint64_t adesc = smem_desc_kmajor_sw128(sa + half * (64 * 128));
                const uint64_t bdesc = smem_desc_kmajor_sw128(sa + kABytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    // +32 bytes per 16 bf16 of K inside the 128-B swizzle atom
                    const int acc_in = ((kb - kb_beg) | k) != 0;
                    if constexpr (BN == 256) wgmma_bf16_ss_n256(acc, adesc + k * 2, bdesc + k * 2, acc_in);
                    else wgmma_bf16_ss_n192(acc, adesc + k * 2, bdesc + k * 2, acc_in);
                }
                wgmma_commit();
                // keep this k-block's MMAs in flight; the previous k-block's have retired -> its stage goes back to the producer
                wgmma_wait<1>();
                reg_fence(acc);
                if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
                prev_s = s;
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
            if (is_unit) {
                const int S = p.sk_splits;
                const int tid = threadIdx.x - 128;  // 0..255 over the two MMA warpgroups
                float* tile_ws = p.sk_ws + (size_t)unit_t * S * (BN / 4) * BM * 4;
                // (1) publish this unit's partial accumulator
                sk_publish<BN>(tile_ws + (size_t)unit_s * (BN / 4) * BM * 4, acc, rit0, c0);
                __threadfence();
                asm volatile("bar.sync 2, 256;" ::: "memory");  // the 8 MMA warps
                // (2) wait until every unit of this tile has published. All units are co-resident: the launch is cooperative
                //     (grid <= SMs x 1 CTA/SM is checked by the runtime), so a unit can only wait for CTAs that are running.
                if (tid == 0) {
                    atomicAdd(p.sk_cnt + 2 * unit_t, 1);
                    uint32_t spins = 0;
                    while (*reinterpret_cast<volatile int*>(p.sk_cnt + 2 * unit_t) < S) {
                        if (++spins > (1u << 26)) __trap();
                    }
                    __threadfence();
                }
                asm volatile("bar.sync 2, 256;" ::: "memory");
                // (3) distributed reduction + fused epilogue on the rows this unit owns (gemm_epilogue.cuh)
                sk_finish<EPI, BN>(p, reinterpret_cast<const float4*>(tile_ws), S, unit_s, m_blk, n_blk, tid);
                // (4) the last unit to finish re-arms the counters for the next launch
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (tid == 0) {
                    const int old = atomicAdd(p.sk_cnt + 2 * unit_t + 1, 1);
                    if (old == S - 1) { p.sk_cnt[2 * unit_t] = 0; p.sk_cnt[2 * unit_t + 1] = 0; }
                }
                break;
            }
            if constexpr (kStaged) {
                // the previous tile has left the staging tile a whole main loop ago; the epilogue warps apply the fused
                // epilogue while this warpgroup runs the next tile's k-blocks
                if constexpr (epi_is_gqa(EPI)) {  // the bias joins the fp32 accumulator before the one bf16 rounding
                    if (p.bias) {
#pragma unroll
                        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const float bv = __bfloat162float(p.bias[n_blk * BN + 8 * j + c0 + e]);
                                acc[4 * j + e] = __fadd_rn(acc[4 * j + e], bv);
                                acc[4 * j + 2 + e] = __fadd_rn(acc[4 * j + 2 + e], bv);
                            }
                    }
                }
                mbar_wait(drained_bar, (it & 1) ^ 1);
                stage_tile<BN>(staging, acc, rit0, c0);
                mbar_arrive(staged_bar);
                ++it;
                last_m = m_blk; last_n = n_blk;
            } else {
                gemm_epilogue_tile<EPI, BN>(p, acc, m_blk, n_blk, rit0, c0);
            }
        }
        if constexpr (kStaged) {
            // this CTA's last tile has no main loop left to hide its epilogue under: the MMA warps drain it together with the
            // epilogue warps once every staging store has landed (a CTA with a split-K unit hides it under the unit instead)
            if (!has_unit && last_m >= 0) {
                mbar_wait(staged_bar, (it - 1) & 1);
                staged_epilogue<EPI, BN>(p, staging, last_m, last_n, kStagedEpiThreads + threadIdx.x - 128, kStagedEpiThreads + 256);
            }
        }
        if constexpr (EPI == EPI_F32) {
            if (p.scat_R > 0) __threadfence_system();  // the pushed rows are visible to their owners before this grid completes
        }
    }
}

// CTA-pair variant (opt-in, MMDP_GEMM_PAIR=1): a cluster of two CTAs computes two m-adjacent 128 x BN tiles of the same n-tile.
// Each CTA loads its own A tile and HALF of the shared W tile, multicast into both CTAs' shared memory, so a pair reads the
// weights once per two m-tiles. A stage is refilled only when the MMA warps of BOTH CTAs have released it (their arrivals
// go to both CTAs' empty barriers). The K loop of every output element is that of gemm_bf16_kernel without a split-K tail:
// the results are bit-identical to it. On one H100 (700 W) the 8B benchmark ran at 70 tokens/s with pairs against 100 with
// the 1-CTA kernel (GEMM time of a sample 16.9 s against 11.0 s), so the 1-CTA kernel is the default.
template <int EPI, int BN>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kGemmThreads, 1)
gemm_pair_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBh, const GemmParams p) {
    constexpr int kStages = GemmCfg<BN, false>::kStages;
    constexpr int kStageBytes = GemmCfg<BN, false>::kStageBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
    uint64_t* empty_bar = full_bar + kStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const uint32_t rank = cluster_ctarank();

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmBh);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 16);  // one arrive per MMA warp of both CTAs
        }
        fence_barrier_init();
    }
    cluster_sync();  // the peer's barriers are initialised before any multicast or remote arrive reaches them
    pdl_launch_dependents();
    pdl_wait();

    const int num_m = (p.M + BM - 1) / BM;
    const int num_n = (p.N + BN - 1) / BN;
    const int num_k = (p.K + BK - 1) / BK;
    const int num_pm = (num_m + 1) / 2;
    const int pair_tiles = num_pm * num_n;
    const int cid = blockIdx.x / 2, n_clusters = gridDim.x / 2;

    if (wg == 0) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one_sync()) {
            int s = 0;
            uint32_t ph = 0;
            for (int t = cid; t < pair_tiles; t += n_clusters) {
                int pm, n_blk;
                gemm_tile_coords(t, num_pm, num_n, p.group_m, pm, n_blk);
                const int m_blk = 2 * pm + (int)rank;  // may be num_m for an odd count: rows read as zero, nothing is stored
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], kStageBytes);
                    uint8_t* sa = smem + s * kStageBytes;
                    tma_load_2d(sa, &tmA, &full_bar[s], kb * BK, m_blk * BM);
                    tma_load_2d_multicast(sa + kABytes + rank * (BN / 2) * 128, &tmBh, &full_bar[s], kb * BK,
                                          n_blk * BN + (int)rank * (BN / 2), 0x3);
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
        }
        __syncwarp();
    } else {
        // ===================== MMA + epilogue =====================
        setmaxnreg_inc<232>();
        const int half = wg - 1;
        const int rit0 = half * 64 + (warp & 3) * 16 + (lane >> 2);
        const int c0 = 2 * (lane & 3);
        float acc[BN / 2];
        int s = 0;
        uint32_t ph = 0;
        for (int t = cid; t < pair_tiles; t += n_clusters) {
            int pm, n_blk;
            gemm_tile_coords(t, num_pm, num_n, p.group_m, pm, n_blk);
            const int m_blk = 2 * pm + (int)rank;
            int prev_s = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(&full_bar[s], ph);
                const uint32_t sa = smem_u32(smem + s * kStageBytes);
                const uint64_t adesc = smem_desc_kmajor_sw128(sa + half * (64 * 128));
                const uint64_t bdesc = smem_desc_kmajor_sw128(sa + kABytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    if constexpr (BN == 256) wgmma_bf16_ss_n256(acc, adesc + k * 2, bdesc + k * 2, (kb | k) != 0);
                    else wgmma_bf16_ss_n192(acc, adesc + k * 2, bdesc + k * 2, (kb | k) != 0);
                }
                wgmma_commit();
                wgmma_wait<1>();
                reg_fence(acc);
                if (prev_s >= 0 && lane == 0) { mbar_arrive(&empty_bar[prev_s]); mbar_arrive_cluster(&empty_bar[prev_s], rank ^ 1u); }
                prev_s = s;
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            if (prev_s >= 0 && lane == 0) { mbar_arrive(&empty_bar[prev_s]); mbar_arrive_cluster(&empty_bar[prev_s], rank ^ 1u); }
            gemm_epilogue_tile<EPI, BN>(p, acc, m_blk, n_blk, rit0, c0);
        }
        if constexpr (EPI == EPI_F32) {
            if (p.scat_R > 0) __threadfence_system();
        }
    }
    cluster_sync();  // neither CTA exits while the other may still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static bool g_coop_pdl_ok = true;  // cleared if the driver rejects cooperative + programmatic launch together

template <int EPI, int BN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int grid, cudaStream_t stream) {
    constexpr int kSmem = GemmCfg<BN, gemm_staged<EPI>()>::kSmem;
    static unsigned long long attr_set = 0;  // bit per device
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    if (!(attr_set >> (dev & 63) & 1ull)) {
        MMDP_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
        attr_set |= 1ull << (dev & 63);
    }
    LaunchScope ls(LK_GEMM, 2.0 * p.M * (double)p.N * p.K, stream);
    // A launch with a split-K tail spin-waits between CTAs -> cooperative launch (the runtime guarantees co-residency of
    // the whole grid or fails the launch; a plain launch could hang behind a concurrent kernel that holds SMs).
    const bool coop = p.sk_tail > 0;
    const bool pdl = pdl_mode() != 0;
    cudaError_t e = launch_ex(gemm_bf16_kernel<EPI, BN>, dim3(grid), dim3(kGemmThreads), kSmem, stream,
                              pdl && (!coop || g_coop_pdl_ok), coop, tmA, tmB, p);
    if (e != cudaSuccess && coop && pdl && g_coop_pdl_ok) {
        (void)cudaGetLastError();
        g_coop_pdl_ok = false;
        e = launch_ex(gemm_bf16_kernel<EPI, BN>, dim3(grid), dim3(kGemmThreads), kSmem, stream, false, true, tmA, tmB, p);
    }
    if (e != cudaSuccess) return set_error("gemm launch failed: %s", cudaGetErrorString(e));
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// Launch plan: tile width (256 | 192), grid, and the split-K tail. Cost model = tile width x (full waves + tail), where a
// split tail costs 1/splits of a wave plus the partial-sum exchange. Split-K changes the fp32 summation ORDER of the
// affected tiles (not the rounding points); which tiles are affected depends on (M, N, K) only, so results are
// deterministic for a given problem shape. MMDP_GEMM_SPLITK: 0 = never, 1 = residual GEMMs only (round-1 behaviour),
// 2 (default) = every epilogue where the cost model says it pays, 3 = every epilogue whenever a tail exists (tests).
struct GemmPlan { int bn, grid, tail, splits, kb_per; };
int gemm_splitk_mode() { return opt(OPT_GEMM_SPLITK); }
void set_gemm_splitk_mode(int m) { set_opt("gemm_splitk", m); }

static GemmPlan plan_gemm(int epi, int M, int N, int K) {
    const int mode = gemm_splitk_mode();
    const int g = num_sms();
    const int num_k = (K + BK - 1) / BK;
    const bool flexible = epi == EPI_PLAIN || epi == EPI_RESID || epi == EPI_F32;
    const bool may_split = num_k >= 4 && (mode >= 2 || (mode == 1 && epi == EPI_RESID));
    GemmPlan best{256, 0, 0, 0, 0};
    double best_cost = 1e30;
    for (int bn : {256, 192}) {
        if (bn == 192 && !flexible) continue;
        const int tiles = ((M + BM - 1) / BM) * ((N + bn - 1) / bn);
        GemmPlan pl{bn, tiles < g ? tiles : g, 0, 0, 0};
        double waves;
        const int full = tiles >= g ? (tiles / g) * g : 0;
        const int tail = tiles - full;
        waves = (double)((tiles + g - 1) / g);
        if (may_split && tail > 0 && tail * 2 <= g) {
            int splits = g / tail;
            if (splits > num_k / 2) splits = num_k / 2;
            if (splits > kSkMaxSplits) splits = kSkMaxSplits;
            if (splits >= 2) {
                const int kb_per = (num_k + splits - 1) / splits;
                splits = (num_k + kb_per - 1) / kb_per;
                // exchange cost in units of one tile's main loop: publish + finish move 2 x 128 KB per unit through L2
                // (~4 us) against num_k x ~0.3 us of MMA time
                const double exch = mode >= 3 ? 0.0 : 12.0 / num_k + 0.04;  // mode 3 (tests): split whenever structurally possible
                const double split_waves = (double)(full / g) + (double)kb_per / num_k + exch;
                if (split_waves < waves) {
                    pl.tail = tail; pl.splits = splits; pl.kb_per = kb_per;
                    pl.grid = full > 0 ? g : tail * splits;
                    waves = split_waves;
                }
            }
        }
        const double cost = waves * bn * (bn == 192 ? 1.04 : 1.0);
        if (cost < best_cost) { best_cost = cost; best = pl; }
    }
    return best;
}

// Split-K workspace: one per (device, stream) - two streams running split GEMMs at the same time must not share partial
// sums or arrival counters. 256 units (>= SMs) x 128 KB + counters, allocated on first use, kept for the life of the process.
struct SkWorkspace { float* ws; int* cnt; };
static std::map<std::pair<int, cudaStream_t>, SkWorkspace> g_sk;
static std::mutex g_sk_mu;
static int splitk_workspace(cudaStream_t stream, SkWorkspace* out) {
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_sk_mu);
    auto key = std::make_pair(dev, stream);
    auto it = g_sk.find(key);
    if (it != g_sk.end()) { *out = it->second; return 0; }
    const size_t units = 256;  // >= number of SMs
    SkWorkspace w{nullptr, nullptr};
    MMDP_CUDA(cudaMalloc(&w.ws, units * BM * 256 * sizeof(float)));
    MMDP_CUDA(cudaMalloc(&w.cnt, 2 * units * sizeof(int)));  // [tile][arrived, finished]
    MMDP_CUDA(cudaMemsetAsync(w.cnt, 0, 2 * units * sizeof(int), stream));
    g_sk.emplace(key, w);
    *out = w;
    return 0;
}

// CTA-pair launch: grid = 2 x the clusters that fit at once (1 CTA per SM; a GPC with an odd SM count leaves one SM out)
template <int EPI, int BN>
static int launch_gemm_pair(const CUtensorMap& tmA, const CUtensorMap& tmBh, const GemmParams& p, int pair_tiles, cudaStream_t stream) {
    static int max_clusters[64] = {0};
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    int& mc = max_clusters[dev & 63];
    if (mc == 0) {
        MMDP_CUDA(cudaFuncSetAttribute(gemm_pair_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN, false>::kSmem));
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(2 * num_sms());
        cfg.blockDim = dim3(kGemmThreads);
        cfg.dynamicSmemBytes = GemmCfg<BN, false>::kSmem;
        cudaLaunchAttribute at{};
        at.id = cudaLaunchAttributeClusterDimension;
        at.val.clusterDim.x = 2; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
        cfg.attrs = &at;
        cfg.numAttrs = 1;
        MMDP_CUDA(cudaOccupancyMaxActiveClusters(&mc, gemm_pair_kernel<EPI, BN>, &cfg));
        if (mc < 1) return set_error("gemm_pair: no cluster of two CTAs fits on this device");
    }
    const int clusters = pair_tiles < mc ? pair_tiles : mc;
    LaunchScope ls(LK_GEMM, 2.0 * p.M * (double)p.N * p.K, stream);
    MMDP_CUDA(launch_ex(gemm_pair_kernel<EPI, BN>, dim3(2 * clusters), dim3(kGemmThreads), GemmCfg<BN, false>::kSmem, stream, pdl_mode() != 0,
                        false, tmA, tmBh, p));
    return 0;
}

int gemm_pair_mode() { return opt(OPT_GEMM_PAIR); }
void set_gemm_pair_mode(int on) { set_opt("gemm_pair", (on == 2) ? 2 : (on ? 1 : 0)); }

int gemm_group_m(int M) {
    const int group_m_env = opt(OPT_GEMM_GROUP_M);
    const int num_m = (M + BM - 1) / BM;
    int g = 0;
    if (num_m > 45) {
        const int ngroups = (num_m + 39) / 40;
        g = (num_m + ngroups - 1) / ngroups;
    }
    return group_m_env >= 0 ? group_m_env : g;
}

int gemm_bf16(int epi, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, int M, int N, int K,
              __nv_bfloat16* C, int ldc, const __nv_bfloat16* resid, int ldr, const QkvRopeArgs* qa,
              cudaStream_t stream, const GemmScatter* sc) {
    if (sc && epi != EPI_F32) return set_error("gemm: the scatter epilogue belongs to MMDP_EPI_F32");
    if (sc && (sc->rows_per_rank <= 0 || sc->slot < 0 || sc->slot > 7 || (M + sc->rows_per_rank - 1) / sc->rows_per_rank > 8))
        return set_error("gemm: bad scatter layout");
    if (M <= 0 || N <= 0 || K <= 0) return set_error("gemm: empty problem");
    if ((lda % 8) || (ldw % 8) || (K % 8)) return set_error("gemm: lda/ldw/K must be multiples of 8 (16-byte TMA strides)");
    if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
        return set_error("gemm: A/W must be 16-byte aligned");
    // argument validation common to both kernels
    switch (epi) {
        case EPI_PLAIN:
            if (!C || (ldc % 8) || (N % 8)) return set_error("gemm: C null or ldc/N not multiple of 8");
            break;
        case EPI_RESID:
            if (!C || !resid || (ldc % 8) || (ldr % 8) || (N % 8)) return set_error("gemm: bad residual epilogue args");
            break;
        case EPI_F32:
            if ((!C && !sc) || (ldc % 4) || (N % 4)) return set_error("gemm: fp32 output needs ldc/N multiples of 4");
            break;
        case EPI_SWIGLU:
            if (!C || (ldc % 8) || (N % 256)) return set_error("gemm: swiglu needs N % 256 == 0 (interleaved gate/up tiles)");
            break;
        case EPI_QKVROPE:
        case EPI_QKVROPE_PACKED:
            if (!qa) return set_error("gemm: qkv epilogue needs QkvRopeArgs");
            if (qa->d_model % 256 || N != 3 * qa->d_model || qa->d_model != qa->n_heads * 128)
                return set_error("gemm: qkv epilogue needs head_dim 128, d_model % 256 == 0, N == 3*d_model");
            if (epi == EPI_QKVROPE_PACKED ? !qa->seg_pos : (qa->pos_map ? (qa->Tq <= 0 || M % qa->Tq) : (!qa->chunked && (M % qa->L))))
                return set_error("gemm: qkv epilogue needs M == B*L (or B*Tq with a position map, or a packed row map)");
            break;
        case EPI_QKVGQA:
        case EPI_QKVGQA_PACKED:
            if (qkv_gqa_check("gemm", epi, M, N, qa)) return -1;
            break;
        default:
            return set_error("gemm: unknown epilogue");
    }
    GemmParams p{};
    p.M = M; p.N = N; p.K = K;
    p.C = C; p.ldc = ldc; p.resid = resid; p.ldr = ldr;
    GemmPlan pl = plan_gemm(epi, M, N, K);
    if (qa && qa->pos_map && pl.tail > 0) {  // the split-K finishing pass addresses rows by sequence position only
        pl.tail = 0; pl.splits = 0; pl.kb_per = 0;
        const int t = ((M + BM - 1) / BM) * ((N + pl.bn - 1) / pl.bn);
        pl.grid = t < num_sms() ? t : num_sms();
    }
    if (sc) {
        // the split-K tail finishes its tiles from the workspace into C; the scatter epilogue has no C - keep whole tiles
        if (pl.tail > 0) { pl.tail = 0; pl.splits = 0; pl.kb_per = 0; const int t = ((M + BM - 1) / BM) * ((N + pl.bn - 1) / pl.bn); pl.grid = t < num_sms() ? t : num_sms(); }
        for (int r = 0; r < 8; ++r) p.scat_dst[r] = sc->dst[r];
        p.scat_R = sc->rows_per_rank; p.scat_slot = sc->slot;
    }
    const int bn = pl.bn, grid = pl.grid;
    // tile order (gemm_tile_coords): with many m-tiles, walk them in balanced groups of <= 40 so that one wave of tiles
    // spans ~30 m-tiles x a few n-tiles instead of all m-tiles x 2-3 n-tiles, which keeps the wave's A rows in L2 while the
    // weights stream (M = 7242: 57 m-tiles, the B=3 batch of a caller that batches its CFG branches); below ~45 m-tiles
    // the plain order is kept (M = 2414). MMDP_GEMM_GROUP_M overrides: 0 = off, n > 0 = fixed group size.
    p.group_m = gemm_group_m(M);
    if (qa) {
        p.q = qa->q; p.k = qa->k; p.vt = qa->vt; p.cos_tab = qa->cos_tab; p.sin_tab = qa->sin_tab;
        p.L = qa->L; p.Lpad = qa->Lpad; p.d_model = qa->d_model; p.n_heads = qa->n_heads;
        p.pos_map = qa->pos_map; p.Tq = qa->Tq; p.row0 = qa->row0; p.seg_pos = qa->seg_pos;
        p.n_kv_heads = qa->n_kv_heads; p.bias = qa->bias;
    }
    // kernel selection: MMDP_GEMM_PAIR / mmdp_set_gemm_pair 0 (default) = one CTA per tile (with the split-K tail), 1 = CTA
    // pairs for M > 256, 2 = pairs only for M >= 4096 and N >= 8192
    const int pmode = gemm_pair_mode();
    if ((pmode == 1 && M > 256) || (pmode == 2 && M >= 4096 && N >= 8192)) {
        p.group_m = (p.group_m + 1) / 2;  // the tile order walks m-tile PAIRS
        const int pair_tiles = ((M + 2 * BM - 1) / (2 * BM)) * ((N + 255) / 256);
        CUtensorMap tmA, tmBh;
        if (make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BM, BK)) return -1;
        if (make_tmap_2d_bf16(&tmBh, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, 128, BK)) return -1;
        switch (epi) {
            case EPI_PLAIN: return launch_gemm_pair<EPI_PLAIN, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_RESID: return launch_gemm_pair<EPI_RESID, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_F32: return launch_gemm_pair<EPI_F32, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_SWIGLU: return launch_gemm_pair<EPI_SWIGLU, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_QKVROPE: return launch_gemm_pair<EPI_QKVROPE, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_QKVROPE_PACKED: return launch_gemm_pair<EPI_QKVROPE_PACKED, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_QKVGQA: return launch_gemm_pair<EPI_QKVGQA, 256>(tmA, tmBh, p, pair_tiles, stream);
            case EPI_QKVGQA_PACKED: return launch_gemm_pair<EPI_QKVGQA_PACKED, 256>(tmA, tmBh, p, pair_tiles, stream);
            default: return set_error("gemm: unknown epilogue");
        }
    }
    if (pl.tail > 0) {
        SkWorkspace w;
        if (splitk_workspace(stream, &w)) return -1;
        p.sk_tail = pl.tail; p.sk_splits = pl.splits; p.sk_kb_per = pl.kb_per; p.sk_ws = w.ws; p.sk_cnt = w.cnt;
    }
    {
        // L2 prefetch of weight tiles: MMDP_GEMM_L2PF = distance in k-blocks (0 = off), MMDP_GEMM_L2PF_MOD = every n-th m-tile
        p.l2pf = opt(OPT_GEMM_L2PF);
        p.l2pf_mod = opt(OPT_GEMM_L2PF_MOD) < 1 ? 1 : opt(OPT_GEMM_L2PF_MOD);
    }
    CUtensorMap tmA, tmB;
    if (make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BM, BK)) return -1;
    if (make_tmap_2d_bf16(&tmB, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, bn, BK)) return -1;
    switch (epi) {
        case EPI_PLAIN:
            return bn == 192 ? launch_gemm<EPI_PLAIN, 192>(tmA, tmB, p, grid, stream) : launch_gemm<EPI_PLAIN, 256>(tmA, tmB, p, grid, stream);
        case EPI_RESID:
            return bn == 192 ? launch_gemm<EPI_RESID, 192>(tmA, tmB, p, grid, stream) : launch_gemm<EPI_RESID, 256>(tmA, tmB, p, grid, stream);
        case EPI_F32:
            return bn == 192 ? launch_gemm<EPI_F32, 192>(tmA, tmB, p, grid, stream) : launch_gemm<EPI_F32, 256>(tmA, tmB, p, grid, stream);
        case EPI_SWIGLU:
            return launch_gemm<EPI_SWIGLU, 256>(tmA, tmB, p, grid, stream);
        case EPI_QKVROPE:
            return launch_gemm<EPI_QKVROPE, 256>(tmA, tmB, p, grid, stream);
        case EPI_QKVROPE_PACKED:
            return launch_gemm<EPI_QKVROPE_PACKED, 256>(tmA, tmB, p, grid, stream);
        case EPI_QKVGQA:
            return launch_gemm<EPI_QKVGQA, 256>(tmA, tmB, p, grid, stream);
        case EPI_QKVGQA_PACKED:
            return launch_gemm<EPI_QKVGQA_PACKED, 256>(tmA, tmB, p, grid, stream);
        default:
            return set_error("gemm: unknown epilogue");
    }
}

}  // namespace mmdp
