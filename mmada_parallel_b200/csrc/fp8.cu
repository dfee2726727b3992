// Opt-in FP8 (e4m3) path of the four linear layers of a block: the quantiser and the persistent e4m3 GEMM for sm_90a.
//
// Quantiser (one definition for weights and activations): for a bf16 row group x[r, gG : (g+1)G]
//   s[g][r] = amax|x| / 448 (fp32, IEEE division; 1 for an all-zero group),  q = e4m3_rn_satfinite(x / s)
// Weights use G = K (one scale per output row), activations G = 128 (a 1 x 128 group per row and k-block).
//
// GEMM: acc[m, n] = sw[n] * sum_g sa[g][m] * (sum_{k in g} qa[m, k] * qw[n, k]), then the fused bf16 epilogues of
// gemm_epilogue.cuh. Same structure as the bf16 kernel (gemm.cu): warpgroup 0 = TMA producer, warpgroups 1 and 2 = wgmma
// on one 64-row half each of a 128 x 128 tile. A k-block is 128 e4m3 = 128 bytes per row, so the 128B-swizzled stage
// layout and the smem descriptors are those of the bf16 kernel. The four m64n128k32 MMAs of a k-block accumulate into a
// fresh fragment that is then promoted into the fp32 master accumulator with the activation scale (the fp8 wgmma
// accumulator keeps fewer bits than fp32; the promotion bounds that error to one k-block). Two 64-register fragments per
// thread are why the tile is 128 wide. No split-K tail and no CTA-pair variant: every tile runs its whole K loop.
// EPI_F32 (tensor-parallel partial sums of the row-parallel linears) stores the scaled fp32 accumulators, or pushes each row to
// the rank that owns it (GemmScatter; gemm_epilogue_tile decides the owner per row, so a 128-row tile may span two owners).
#include "gemm_epilogue.cuh"

namespace mmdp {

// ------------------------------------------------------------------------------------------------
// quantiser: one warp per (row, group) with lane l holding elements 4l + 128t of the group; for the activation groups
// (G = 128) one half-warp per group with 16-byte loads, so that twice the bytes per thread are in flight
// ------------------------------------------------------------------------------------------------
// (absmax4 / quant4: ptx.cuh)
__global__ void __launch_bounds__(256) quantize_fp8_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int rows, int K, int G,
                                                           uint8_t* __restrict__ q, int ldq, float* __restrict__ scales) {
    const int ng = K / G;
    const long long item = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    pdl_launch_dependents();
    pdl_wait();
    if (item >= (long long)rows * ng) return;
    const int r = (int)(item / ng), g = (int)(item - (long long)r * ng);
    const __nv_bfloat16* src = x + (size_t)r * ldx + (size_t)g * G + 4 * lane;
    uint8_t* dst = q + (size_t)r * ldq + (size_t)g * G + 4 * lane;
    float amax = 0.f;
    for (int t = 0; t < G / 128; ++t) amax = absmax4(*reinterpret_cast<const uint2*>(src + 128 * t), amax);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float s = amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f;
    for (int t = 0; t < G / 128; ++t)
        *reinterpret_cast<uint32_t*>(dst + 128 * t) = quant4(*reinterpret_cast<const uint2*>(src + 128 * t), s);
    if (lane == 0) scales[(size_t)g * rows + r] = s;
}

// G = 128, x / q rows 16- / 8-byte aligned: half-warp h of a warp takes group 2 w + h, lane l of it elements 8l .. 8l + 7
__global__ void __launch_bounds__(256) quantize_fp8_g128_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int rows, int ng,
                                                                uint8_t* __restrict__ q, int ldq, float* __restrict__ scales) {
    const long long item = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * 2 + ((threadIdx.x >> 4) & 1);
    const int l = threadIdx.x & 15;
    const unsigned half_mask = 0xffffu << (threadIdx.x & 16);
    pdl_launch_dependents();
    pdl_wait();
    if (item >= (long long)rows * ng) return;
    const int r = (int)(item / ng), g = (int)(item - (long long)r * ng);
    const uint4 v = *reinterpret_cast<const uint4*>(x + (size_t)r * ldx + (size_t)g * 128 + 8 * l);
    const uint2 v0 = make_uint2(v.x, v.y), v1 = make_uint2(v.z, v.w);
    float amax = absmax4(v1, absmax4(v0, 0.f));
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(half_mask, amax, o));
    const float s = amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f;
    *reinterpret_cast<uint2*>(q + (size_t)r * ldq + (size_t)g * 128 + 8 * l) = make_uint2(quant4(v0, s), quant4(v1, s));
    if (l == 0) scales[(size_t)g * rows + r] = s;
}

int quantize_fp8(const __nv_bfloat16* x, int ldx, int rows, int K, int group, uint8_t* q, int ldq, float* scales,
                 cudaStream_t stream) {
    if (rows <= 0) return 0;
    if (!x || !q || !scales) return set_error("quantize_fp8: null argument");
    if (K <= 0 || group <= 0 || group % 128 || K % group) return set_error("quantize_fp8: group must be a multiple of 128 that divides K (K=%d, group=%d)", K, group);
    if (ldx < K || ldq < K || (ldx % 4) || (ldq % 4)) return set_error("quantize_fp8: ldx/ldq must be >= K and multiples of 4");
    if ((reinterpret_cast<uintptr_t>(x) & 7) || (reinterpret_cast<uintptr_t>(q) & 3)) return set_error("quantize_fp8: x must be 8-byte, q 4-byte aligned");
    const long long items = (long long)rows * (K / group);
    LaunchScope ls(LK_ROW, (double)rows * K * 3 + 4.0 * items, stream);  // bytes: read bf16, write e4m3 + scales
    const bool g128 = group == 128 && !(ldx % 8) && !(ldq % 8) && !(reinterpret_cast<uintptr_t>(x) & 15) && !(reinterpret_cast<uintptr_t>(q) & 7);
    if (g128)
        MMDP_CUDA(launch_ex(quantize_fp8_g128_kernel, dim3((unsigned)((items + 15) / 16)), dim3(256), 0, stream, pdl_mode() != 0, false, x,
                            ldx, rows, K / 128, q, ldq, scales));
    else
        MMDP_CUDA(launch_ex(quantize_fp8_kernel, dim3((unsigned)((items + 7) / 8)), dim3(256), 0, stream, pdl_mode() != 0, false, x, ldx,
                            rows, K, group, q, ldq, scales));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// e4m3 GEMM
// ------------------------------------------------------------------------------------------------
static constexpr int kF8BM = 128, kF8BN = 128, kF8BK = 128;  // BK in e4m3 elements (= bytes)
static constexpr int kF8TileBytes = kF8BM * kF8BK;           // 16 KB (A and W tiles alike)
static constexpr int kF8StageBytes = 2 * kF8TileBytes;
static constexpr int kF8Stages = 6;                          // 192 KB of the 227 KB an H100 block may use
static constexpr int kF8Smem = kF8Stages * kF8StageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static constexpr int kF8Threads = 384;

struct Fp8Scales {
    const float* sa;  // [K / 128][M]
    const float* sw;  // [N]
};

template <int EPI>
__global__ void __launch_bounds__(kF8Threads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p, const Fp8Scales sc) {
    constexpr int BN = kF8BN;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kF8Stages * kF8StageBytes);
    uint64_t* empty_bar = full_bar + kF8Stages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kF8Stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrive per MMA warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    const int num_m = (p.M + kF8BM - 1) / kF8BM;
    const int num_n = (p.N + BN - 1) / BN;
    const int num_k = p.K / kF8BK;
    const int num_tiles = num_m * num_n;

    if (wg == 0) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one_sync()) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int m_blk, n_blk;
                gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], kF8StageBytes);
                    uint8_t* st = smem + s * kF8StageBytes;
                    tma_load_2d(st, &tmA, &full_bar[s], kb * kF8BK, m_blk * kF8BM);
                    tma_load_2d(st + kF8TileBytes, &tmB, &full_bar[s], kb * kF8BK, n_blk * BN);
                    if (++s == kF8Stages) { s = 0; ph ^= 1; }
                }
            }
        }
        __syncwarp();
    } else {
        // ===================== MMA + promotion + epilogue (warpgroups 1 and 2: tile rows [64 (wg-1), 64 wg)) =====================
        setmaxnreg_inc<232>();
        const int half = wg - 1;
        const int rit0 = half * 64 + (warp & 3) * 16 + (lane >> 2);  // tile row of acc[4j + 0..1]; acc[4j + 2..3] is 8 rows below
        const int c0 = 2 * (lane & 3);
        float acc[BN / 2], part[BN / 2];
        int s = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int m_blk, n_blk;
            gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
            const int row0 = m_blk * kF8BM + rit0, row1 = row0 + 8;
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(&full_bar[s], ph);
                const uint32_t st = smem_u32(smem + s * kF8StageBytes);
                const uint64_t adesc = smem_desc_kmajor_sw128(st + half * (64 * 128));
                const uint64_t bdesc = smem_desc_kmajor_sw128(st + kF8TileBytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kF8BK / 32; ++k)  // +32 bytes per 32 e4m3 of K inside the 128-B swizzle atom
                    wgmma_e4m3_ss_n128(part, adesc + k * 2, bdesc + k * 2, k != 0);
                wgmma_commit();
                // this k-block's activation scales of the thread's two rows; the loads overlap the MMAs
                const float* sak = sc.sa + (size_t)kb * p.M;
                const float s0 = row0 < p.M ? __ldg(sak + row0) : 0.f;
                const float s1 = row1 < p.M ? __ldg(sak + row1) : 0.f;
                wgmma_wait<0>();
                reg_fence(part);
                if (lane == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] = fmaf(part[i], (i & 2) ? s1 : s0, acc[i]);
                if (++s == kF8Stages) { s = 0; ph ^= 1; }
            }
            // weight row scales (columns of the tile), once per tile
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = n_blk * BN + 8 * j + c0;
                const float w0 = col < p.N ? __ldg(sc.sw + col) : 0.f;
                const float w1 = col + 1 < p.N ? __ldg(sc.sw + col + 1) : 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    acc[4 * j + 2 * h] = __fmul_rn(acc[4 * j + 2 * h], w0);
                    acc[4 * j + 2 * h + 1] = __fmul_rn(acc[4 * j + 2 * h + 1], w1);
                }
            }
            gemm_epilogue_tile<EPI, BN>(p, acc, m_blk, n_blk, rit0, c0);
        }
        if constexpr (EPI == EPI_F32) {
            if (p.scat_R > 0) __threadfence_system();  // the pushed rows are visible to their owners before this grid completes
        }
    }
}

template <int EPI>
static int launch_gemm_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, const Fp8Scales& sc, int grid,
                           cudaStream_t stream) {
    static unsigned long long attr_set = 0;  // bit per device
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    if (!(attr_set >> (dev & 63) & 1ull)) {
        MMDP_CUDA(cudaFuncSetAttribute(gemm_fp8_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kF8Smem));
        attr_set |= 1ull << (dev & 63);
    }
    LaunchScope ls(LK_GEMM, 2.0 * p.M * (double)p.N * p.K, stream);
    MMDP_CUDA(launch_ex(gemm_fp8_kernel<EPI>, dim3(grid), dim3(kF8Threads), kF8Smem, stream, pdl_mode() != 0, false, tmA, tmB, p, sc));
    return 0;
}

int gemm_fp8(int epi, const uint8_t* A, int lda, const float* sa, const uint8_t* W, int ldw, const float* sw, int M, int N,
             int K, __nv_bfloat16* C, int ldc, const __nv_bfloat16* resid, int ldr, const QkvRopeArgs* qa, cudaStream_t stream,
             const GemmScatter* scat) {
    if (scat && epi != EPI_F32) return set_error("gemm_fp8: the scatter epilogue belongs to EPI_F32");
    if (scat && (scat->rows_per_rank <= 0 || scat->slot < 0 || scat->slot > 7 || (M + scat->rows_per_rank - 1) / scat->rows_per_rank > 8))
        return set_error("gemm_fp8: bad scatter layout");
    if (M <= 0 || N <= 0 || K <= 0) return set_error("gemm_fp8: empty problem");
    if (!A || !W || !sa || !sw) return set_error("gemm_fp8: null operand or scale pointer");
    if (K % kF8BK) return set_error("gemm_fp8: K must be a multiple of 128 (the activation scale group)");
    if ((lda % 16) || (ldw % 16)) return set_error("gemm_fp8: lda/ldw must be multiples of 16 (16-byte TMA strides)");
    if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(W) & 15)) return set_error("gemm_fp8: A/W must be 16-byte aligned");
    switch (epi) {
        case EPI_PLAIN:
            if (!C || (ldc % 8) || (N % 8)) return set_error("gemm_fp8: C null or ldc/N not multiple of 8");
            break;
        case EPI_RESID:
            if (!C || !resid || (ldc % 8) || (ldr % 8) || (N % 8)) return set_error("gemm_fp8: bad residual epilogue args");
            break;
        case EPI_F32:
            if ((!C && !scat) || (ldc % 4) || (N % 4)) return set_error("gemm_fp8: fp32 output needs ldc/N multiples of 4");
            break;
        case EPI_SWIGLU:
            if (!C || (ldc % 8) || (N % kF8BN)) return set_error("gemm_fp8: swiglu needs N %% 128 == 0 (gate/up interleaved in 64-row blocks)");
            break;
        case EPI_QKVROPE:
        case EPI_QKVROPE_PACKED:
            if (!qa) return set_error("gemm_fp8: qkv epilogue needs QkvRopeArgs");
            if (qa->d_model % 256 || N != 3 * qa->d_model || qa->d_model != qa->n_heads * 128)
                return set_error("gemm_fp8: qkv epilogue needs head_dim 128, d_model %% 256 == 0, N == 3*d_model");
            if (epi == EPI_QKVROPE_PACKED ? !qa->seg_pos : (qa->pos_map ? (qa->Tq <= 0 || M % qa->Tq) : (!qa->chunked && (M % qa->L))))
                return set_error("gemm_fp8: qkv epilogue needs M == B*L (or B*Tq with a position map, or a packed row map)");
            break;
        case EPI_QKVGQA:
        case EPI_QKVGQA_PACKED:
            if (qkv_gqa_check("gemm_fp8", epi, M, N, qa)) return -1;
            break;
        default:
            return set_error("gemm_fp8: unsupported epilogue %d", epi);
    }
    GemmParams p{};
    p.M = M; p.N = N; p.K = K;
    p.C = C; p.ldc = ldc; p.resid = resid; p.ldr = ldr;
    p.group_m = gemm_group_m(M);
    if (qa) {
        p.q = qa->q; p.k = qa->k; p.vt = qa->vt; p.cos_tab = qa->cos_tab; p.sin_tab = qa->sin_tab;
        p.L = qa->L; p.Lpad = qa->Lpad; p.d_model = qa->d_model; p.n_heads = qa->n_heads;
        p.pos_map = qa->pos_map; p.Tq = qa->Tq; p.row0 = qa->row0; p.seg_pos = qa->seg_pos;
        p.n_kv_heads = qa->n_kv_heads; p.bias = qa->bias;
    }
    if (scat) {
        for (int r = 0; r < 8; ++r) p.scat_dst[r] = scat->dst[r];
        p.scat_R = scat->rows_per_rank; p.scat_slot = scat->slot;
    }
    const Fp8Scales sc{sa, sw};
    const int tiles = ((M + kF8BM - 1) / kF8BM) * ((N + kF8BN - 1) / kF8BN);
    const int grid = tiles < num_sms() ? tiles : num_sms();
    CUtensorMap tmA, tmB;
    if (make_tmap_2d(&tmA, A, 1, (uint64_t)M, (uint64_t)K, (uint64_t)lda, kF8BM, kF8BK)) return -1;
    if (make_tmap_2d(&tmB, W, 1, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, kF8BN, kF8BK)) return -1;
    switch (epi) {
        case EPI_PLAIN: return launch_gemm_fp8<EPI_PLAIN>(tmA, tmB, p, sc, grid, stream);
        case EPI_RESID: return launch_gemm_fp8<EPI_RESID>(tmA, tmB, p, sc, grid, stream);
        case EPI_F32: return launch_gemm_fp8<EPI_F32>(tmA, tmB, p, sc, grid, stream);
        case EPI_SWIGLU: return launch_gemm_fp8<EPI_SWIGLU>(tmA, tmB, p, sc, grid, stream);
        case EPI_QKVROPE_PACKED: return launch_gemm_fp8<EPI_QKVROPE_PACKED>(tmA, tmB, p, sc, grid, stream);
        case EPI_QKVGQA: return launch_gemm_fp8<EPI_QKVGQA>(tmA, tmB, p, sc, grid, stream);
        case EPI_QKVGQA_PACKED: return launch_gemm_fp8<EPI_QKVGQA_PACKED>(tmA, tmB, p, sc, grid, stream);
        default: return launch_gemm_fp8<EPI_QKVROPE>(tmA, tmB, p, sc, grid, stream);
    }
}

}  // namespace mmdp
