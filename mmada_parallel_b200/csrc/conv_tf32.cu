// TF32 wgmma "shifted-tap" GEMM: the convolution engine of the VQ decoders (MAGVITv2.decode_code,
// MMaDA-Parallel-M/models/modeling_magvitv2.py:365-399,429-433; blocks in models/common_modules.py).
//
//   C[m, n] = bias + sum_{t < T} sum_k A[m + shift[t], k] * W[t*N + n, k]   (+ R[m, n])          fp32 in / fp32 out
//
// Activations are channels-last fp32 with a one-pixel zero border per image ("padded NHWC": row index
// (y+1)*(W+2) + (x+1), C contiguous), so a 3x3 convolution is nine GEMM taps whose A tiles are the SAME activation
// matrix read at nine row offsets - a TMA tile load with a shifted row coordinate (out-of-range rows read as zero).
// All taps accumulate into one register accumulator (K loop = taps x channel blocks); tf32 wgmma consumes the fp32
// tiles directly (10-bit mantissa, what cuDNN does for the reference on a GPU with allow_tf32). 1x1 convolutions and
// the AttnBlock matmuls are the T = 1 case. Same warp-specialised pipeline as gemm.cu (TMA warpgroup, two MMA warpgroups).
#include "mmdp_internal.h"
#include "ptx.cuh"

namespace mmdp {

static constexpr int CBM = 128, CBN = 128, CBK = 32;  // 32 fp32 = one 128-byte swizzle row
static constexpr int kCStages = 6;
static constexpr int kCABytes = CBM * CBK * 4;  // 16 KB
static constexpr int kCBBytes = CBN * CBK * 4;  // 16 KB
static constexpr int kCStageBytes = kCABytes + kCBBytes;
static constexpr int kConvThreads = 384;
static constexpr int kConvSmem = kCStages * kCStageBytes + 1024 + 256;
static constexpr int kMaxTaps = 9;

struct ConvParams {
    int M, N, K;  // rows of the A/C index space, output channels, padded input channels (multiple of 32)
    int T;
    int shift[kMaxTaps];
    float* C;
    int ldc;
    const float* R;  // optional residual, same row space as C
    int ldr;
    const float* bias;  // optional
    int bias_along_m;
    float alpha;  // C = alpha * acc + bias (+ R)
    // row-space handling
    int pad_w, pad_h;  // > 0: rows index a padded image (pad_w = W + 2, pad_h = H + 2); border rows are written as zero
    int scatter_w;     // > 0: rows index a compact W-wide image; C/R rows live in the padded layout of that image
    int scatter_h;
};

__global__ void __launch_bounds__(kConvThreads, 1)
conv_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const ConvParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kCStages * kCStageBytes);
    uint64_t* empty_bar = full_bar + kCStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW);
        for (int s = 0; s < kCStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    const int num_m = (p.M + CBM - 1) / CBM, num_n = (p.N + CBN - 1) / CBN;
    const int kblocks = p.K / CBK;
    const int num_k = p.T * kblocks;
    const int num_tiles = num_m * num_n;

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one_sync()) {
            int s = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int n_blk = tile % num_n, m_blk = tile / num_n;  // n fastest: CTAs running together share the A rows
                for (int kb = 0; kb < num_k; ++kb) {
                    const int t = kb / kblocks, kc = kb - t * kblocks;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], kCStageBytes);
                    uint8_t* sa = smem + s * kCStageBytes;
                    tma_load_2d(sa, &tmA, &full_bar[s], kc * CBK, m_blk * CBM + p.shift[t]);
                    tma_load_2d(sa + kCABytes, &tmW, &full_bar[s], kc * CBK, t * p.N + n_blk * CBN);
                    if (++s == kCStages) { s = 0; ph ^= 1; }
                }
            }
        }
        __syncwarp();
    } else {
        setmaxnreg_inc<232>();
        const int half = wg - 1;
        const int rit0 = half * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
        float acc[CBN / 2];
        int s = 0; uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int n_blk = tile % num_n, m_blk = tile / num_n;
            int prev_s = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(&full_bar[s], ph);
                const uint32_t sa = smem_u32(smem + s * kCStageBytes);
                const uint64_t adesc = smem_desc_kmajor_sw128(sa + half * (64 * 128)), bdesc = smem_desc_kmajor_sw128(sa + kCABytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < CBK / 8; ++k)  // K = 8 per tf32 wgmma: 32 bytes per step inside the swizzle atom
                    wgmma_tf32_ss_n128(acc, adesc + k * 2, bdesc + k * 2, (kb | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();
                reg_fence(acc);
                if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
                prev_s = s;
                if (++s == kCStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = m_blk * CBM + rit0 + 8 * h;
                if (row >= p.M) continue;
                bool interior = true;
                long long orow = row;
                if (p.pad_w > 0) {
                    const int per = p.pad_w * p.pad_h;
                    const int r = row % per;
                    const int y = r / p.pad_w, x = r - y * p.pad_w;
                    interior = (y >= 1) && (y <= p.pad_h - 2) && (x >= 1) && (x <= p.pad_w - 2);
                } else if (p.scatter_w > 0) {
                    const int per = p.scatter_w * p.scatter_h;
                    const int b = row / per, r = row - b * per;
                    const int y = r / p.scatter_w, x = r - y * p.scatter_w;
                    orow = (long long)b * (p.scatter_w + 2) * (p.scatter_h + 2) + (long long)(y + 1) * (p.scatter_w + 2) + (x + 1);
                }
                float* dst = p.C + orow * p.ldc;
                const float* rsd = p.R ? p.R + orow * p.ldr : nullptr;
                const float bm = (p.bias && p.bias_along_m) ? p.bias[row] : 0.f;
#pragma unroll
                for (int j = 0; j < CBN / 8; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = n_blk * CBN + 8 * j + c0 + e;
                        if (col < p.N) {
                            float o = 0.f;
                            if (interior) {
                                o = acc[4 * j + 2 * h + e] * p.alpha;
                                if (p.bias) o += p.bias_along_m ? bm : p.bias[col];
                                if (rsd) o += rsd[col];
                            }
                            dst[col] = o;
                        }
                    }
                }
            }
        }
    }
}

int conv_tf32(const float* A, int lda, long long a_rows, const float* W, int M, int N, int K, int T, const int* shifts,
              float* C, int ldc, const float* R, int ldr, const float* bias, int bias_along_m, float alpha, int pad_w,
              int pad_h, int scatter_w, int scatter_h, cudaStream_t stream) {
    if (M <= 0 || N <= 0 || K <= 0 || T <= 0 || T > kMaxTaps) return set_error("conv_tf32: bad problem size");
    if (K % CBK) return set_error("conv_tf32: K (padded input channels) must be a multiple of 32");
    if (lda % 4) return set_error("conv_tf32: lda must be a multiple of 4 (16-byte TMA stride)");
    ConvParams p{};
    p.M = M; p.N = N; p.K = K; p.T = T;
    for (int t = 0; t < T; ++t) p.shift[t] = shifts ? shifts[t] : 0;
    p.C = C; p.ldc = ldc; p.R = R; p.ldr = ldr; p.bias = bias; p.bias_along_m = bias_along_m; p.alpha = alpha;
    p.pad_w = pad_w; p.pad_h = pad_h; p.scatter_w = scatter_w; p.scatter_h = scatter_h;
    CUtensorMap tmA, tmW;
    if (make_tmap_2d(&tmA, A, 4, (uint64_t)a_rows, (uint64_t)K, (uint64_t)lda, CBM, CBK)) return -1;
    if (make_tmap_2d(&tmW, W, 4, (uint64_t)T * N, (uint64_t)K, (uint64_t)K, CBN, CBK)) return -1;
    static bool attr_set = false;
    if (!attr_set) {
        MMDP_CUDA(cudaFuncSetAttribute(conv_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmem));
        attr_set = true;
    }
    const int num_tiles = ((M + CBM - 1) / CBM) * ((N + CBN - 1) / CBN);
    const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
    LaunchScope ls(LK_GEMM, 2.0 * M * (double)N * K * T, stream);
    conv_tf32_kernel<<<grid, kConvThreads, kConvSmem, stream>>>(tmA, tmW, p);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// row kernels of the decoder (HBM-bound)
// ------------------------------------------------------------------------------------------------
// GroupNorm(32 groups) statistics over the interior pixels of padded NHWC images. grid (chunks, B); thread layout:
// TC = min(C, 256) lanes along channels (coalesced), 256/TC lanes along pixels; fp64 accumulation across CTAs.
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int C, int H, int W, double* __restrict__ stats) {
    // per-(image, group) sum and sum of squares of the interior pixels. A thread owns four consecutive channels (one float4) and
    // walks the CTA's pixel chunk with 256 / (C/4) pixel lanes, four independent loads in flight (the first version - one
    // scalar load per thread and iteration, 256 CTAs - ran at 0.5 TB/s on the 134 MB full-resolution tensors: latency-bound)
    const int b = blockIdx.y, Wp = W + 2, cpg = C / 32, C4 = C / 4;
    const float4* xb = reinterpret_cast<const float4*>(x + (size_t)b * (H + 2) * Wp * C);
    const int TC = C4 < 256 ? C4 : 256, PP = 256 / TC;
    const int cl = threadIdx.x % TC, pl = threadIdx.x / TC;
    const long long npix = (long long)H * W;
    const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
    const long long p0 = (long long)blockIdx.x * chunk;
    const long long p1 = p0 + chunk < npix ? p0 + chunk : npix;
    __shared__ double s_sum[32], s_sq[32];
    if (threadIdx.x < 32) { s_sum[threadIdx.x] = 0.0; s_sq[threadIdx.x] = 0.0; }
    __syncthreads();
    if (pl < PP) {
        for (int c4 = cl; c4 < C4; c4 += TC) {
            float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
            for (long long pp = p0 + pl; pp < p1; pp += 4LL * PP) {
                float4 v[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const long long pt = pp + (long long)t * PP;
                    if (pt < p1) {
                        const int y = (int)(pt / W), xx = (int)(pt - (long long)y * W);
                        v[t] = xb[((size_t)(y + 1) * Wp + xx + 1) * C4 + c4];
                    } else {
                        v[t] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    s[0] += v[t].x; s[1] += v[t].y; s[2] += v[t].z; s[3] += v[t].w;
                    q[0] = fmaf(v[t].x, v[t].x, q[0]); q[1] = fmaf(v[t].y, v[t].y, q[1]);
                    q[2] = fmaf(v[t].z, v[t].z, q[2]); q[3] = fmaf(v[t].w, v[t].w, q[3]);
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                atomicAdd(&s_sum[(c4 * 4 + k) / cpg], (double)s[k]);
                atomicAdd(&s_sq[(c4 * 4 + k) / cpg], (double)q[k]);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        atomicAdd(&stats[((size_t)b * 32 + threadIdx.x) * 2], s_sum[threadIdx.x]);
        atomicAdd(&stats[((size_t)b * 32 + threadIdx.x) * 2 + 1], s_sq[threadIdx.x]);
    }
}

// y = swish?( (x - mean) * rstd * gamma + beta ). compact == 0: padded NHWC out (border pixels are written as zero, so a
// buffer that held another geometry before is valid padding again); compact == 1: [B, H*W, C] out.
__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int H, int W,
                                                        const double* __restrict__ stats, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int swish, int compact) {
    // one CTA per (padded image row, batch image): float4 over the channels, the 32 group means / inverse deviations are
    // evaluated once per CTA (fp64, like the sums they come from), no per-element 64-bit division
    const int b = blockIdx.y, yy = blockIdx.x, Wp = W + 2, Hp = H + 2, cpg = C / 32, C4 = C / 4;
    __shared__ float s_mean[32], s_rstd[32];
    if (threadIdx.x < 32) {
        const double cnt = (double)H * W * cpg;
        const double mean = stats[((size_t)b * 32 + threadIdx.x) * 2] / cnt;
        const double var = stats[((size_t)b * 32 + threadIdx.x) * 2 + 1] / cnt - mean * mean;
        s_mean[threadIdx.x] = (float)mean;
        s_rstd[threadIdx.x] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
    const bool row_in = yy >= 1 && yy <= H;
    const size_t row_base = ((size_t)b * Hp + yy) * Wp;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
    float4* y4 = reinterpret_cast<float4*>(y);
    for (int j = threadIdx.x; j < Wp * C4; j += blockDim.x) {
        const int xx = j / C4, c4 = j - xx * C4;
        const bool interior = row_in && xx >= 1 && xx <= W;
        if (!interior) {
            if (!compact) y4[(row_base + xx) * C4 + c4] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const float4 v = x4[(row_base + xx) * C4 + c4];
        const float4 gm = g4[c4], bt = b4[c4];
        const float in[4] = {v.x, v.y, v.z, v.w}, gg[4] = {gm.x, gm.y, gm.z, gm.w}, bb[4] = {bt.x, bt.y, bt.z, bt.w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int g = (c4 * 4 + k) / cpg;
            float t = (in[k] - s_mean[g]) * s_rstd[g] * gg[k] + bb[k];
            if (swish) t = t / (1.0f + expf(-t));
            o[k] = t;
        }
        const size_t dst = compact ? ((size_t)b * H * W + (size_t)(yy - 1) * W + (xx - 1)) * C4 + c4 : (row_base + xx) * C4 + c4;
        y4[dst] = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// nearest 2x upsample, padded NHWC -> padded NHWC (border of the output written as zero)
__global__ void __launch_bounds__(256) upsample2x_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int H, int W) {
    const int b = blockIdx.y, Wp = W + 2, W2 = 2 * W, H2 = 2 * H, Wp2 = W2 + 2, Hp2 = H2 + 2;
    const int C4 = C / 4;
    const long long n = (long long)Hp2 * Wp2 * C4;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* y4 = reinterpret_cast<float4*>(y);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        const long long pix = i / C4;
        const int yy = (int)(pix / Wp2), xx = (int)(pix - (long long)yy * Wp2);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (yy >= 1 && yy <= H2 && xx >= 1 && xx <= W2)
            v = x4[((size_t)b * (H + 2) * Wp + (size_t)((yy - 1) / 2 + 1) * Wp + (xx - 1) / 2 + 1) * C4 + c];
        y4[(size_t)b * n + i] = v;
    }
}

// in-place row softmax of an fp32 matrix [rows, n]
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ s, int n, int ld) {
    float* row = s + (size_t)blockIdx.x * ld;
    __shared__ float red[8];
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, row[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float e = expf(row[i] - mx); row[i] = e; sum += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = 0.f;
    for (int i = 0; i < 8; ++i) sum += red[i];
    const float inv = 1.0f / sum;
    for (int i = threadIdx.x; i < n; i += blockDim.x) row[i] *= inv;
}

// LFQ codebook entry straight into the padded NHWC input of the decoder: ids [B, H*W] -> z [B, (H+2)(W+2), Cpad] (+-1, rest 0)
__global__ void lfq_to_padded_kernel(const int64_t* __restrict__ ids, float* __restrict__ z, int H, int W, int bits, int Cpad) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= H * W) return;
    const int64_t id = ids[(size_t)b * H * W + n];
    const int y = n / W, x = n - y * W;
    float* dst = z + ((size_t)b * (H + 2) * (W + 2) + (size_t)(y + 1) * (W + 2) + x + 1) * Cpad;
    for (int c = 0; c < bits; ++c) dst[c] = ((id >> (bits - 1 - c)) & 1) ? 1.0f : -1.0f;
}

// padded NHWC [B, (H+2)(W+2), ld] -> NCHW [B, C, H, W]
__global__ void padded_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int ld, int H, int W) {
    const int b = blockIdx.y;
    const long long n = (long long)C * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int xx = (int)(i % W);
        const int yy = (int)((i / W) % H);
        const int c = (int)(i / ((long long)W * H));
        y[(size_t)b * n + i] = x[((size_t)b * (H + 2) * (W + 2) + (size_t)(yy + 1) * (W + 2) + xx + 1) * ld + c];
    }
}

// ---- encoder-side row kernels (MAGVITv2.get_code) ---------------------------------------------------------------
// NCHW pixels [B, C, H, W] -> padded channels-last [B, (H+2)(W+2), Cpad] (extra channels and the border are zero)
__global__ void __launch_bounds__(256) nchw_to_padded_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int Cpad, int H, int W) {
    const int b = blockIdx.y, Wp = W + 2, Hp = H + 2;
    const long long n = (long long)Hp * Wp * Cpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cpad);
        const long long pix = i / Cpad;
        const int yy = (int)(pix / Wp), xx = (int)(pix - (long long)yy * Wp);
        float v = 0.f;
        if (c < C && yy >= 1 && yy <= H && xx >= 1 && xx <= W) v = x[(((size_t)b * C + c) * H + (yy - 1)) * W + (xx - 1)];
        y[(size_t)b * n + i] = v;
    }
}
// Downsample (common_modules.py:73-90): pad (0,1,0,1) + 3x3 stride-2 conv == the stride-1 zero-border conv evaluated at
// input pixel (2y+1, 2x+1). src: padded [B, (H+2)(W+2), C] holding the stride-1 result; dst: padded [B, (H/2+2)(W/2+2), C].
__global__ void __launch_bounds__(256) downsample_pick_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int H, int W) {
    const int b = blockIdx.y, Wp = W + 2, H2 = H / 2, W2 = W / 2, Wp2 = W2 + 2, Hp2 = H2 + 2, C4 = C / 4;
    const long long n = (long long)Hp2 * Wp2 * C4;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        const long long pix = i / C4;
        const int yy = (int)(pix / Wp2), xx = (int)(pix - (long long)yy * Wp2);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (yy >= 1 && yy <= H2 && xx >= 1 && xx <= W2)
            v = s4[((size_t)b * (H + 2) * Wp + (size_t)(2 * (yy - 1) + 2) * Wp + (2 * (xx - 1) + 2)) * C4 + c];
        d4[(size_t)b * n + i] = v;
    }
}
// LFQ sign quantisation + get_indices (modeling_magvitv2.py:201-206): padded [B, (h+2)(w+2), ld] -> int64 ids [B, h*w]
__global__ void lfq_indices_kernel(const float* __restrict__ z, int64_t* __restrict__ ids, int h, int w, int bits, int ld) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= h * w) return;
    const int y = n / w, x = n - y * w;
    const float* src = z + ((size_t)b * (h + 2) * (w + 2) + (size_t)(y + 1) * (w + 2) + x + 1) * ld;
    int64_t id = 0;
    for (int c = 0; c < bits; ++c) id |= (int64_t)(src[c] > 0.f) << (bits - 1 - c);
    ids[(size_t)b * h * w + n] = id;
}

int nchw_to_padded(const float* x, float* y, int B, int C, int Cpad, int H, int W, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * H * W * (C + Cpad) * 4, stream);
    nchw_to_padded_kernel<<<dim3(num_sms() * 4, B), 256, 0, stream>>>(x, y, C, Cpad, H, W);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}
int downsample_pick(const float* src, float* dst, int B, int C, int H, int W, cudaStream_t stream) {
    if ((C % 4) || (H % 2) || (W % 2)) return set_error("downsample: C %% 4 and even H, W required");
    LaunchScope ls(LK_ROW, (double)B * (H / 2) * (W / 2) * C * 8, stream);
    downsample_pick_kernel<<<dim3(num_sms() * 4, B), 256, 0, stream>>>(src, dst, C, H, W);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}
int lfq_indices(const float* z, int64_t* ids, int B, int h, int w, int bits, int ld, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * h * w * (bits * 4 + 8), stream);
    lfq_indices_kernel<<<dim3((h * w + 255) / 256, B), 256, 0, stream>>>(z, ids, h, w, bits, ld);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int gn_swish(const float* x, float* y, int B, int C, int H, int W, double* stats_ws, const float* gamma, const float* beta,
             float eps, int swish, int compact, cudaStream_t stream) {
    if (C % 32) return set_error("group_norm: channels must be a multiple of 32");
    MMDP_CUDA(cudaMemsetAsync(stats_ws, 0, (size_t)B * 32 * 2 * sizeof(double), stream));
    const long long npix = (long long)H * W;
    int chunks = (int)((npix + 127) / 128);
    if (chunks > num_sms() * 16) chunks = num_sms() * 16;
    {
        LaunchScope ls(LK_ROW, (double)B * npix * C * 4, stream);
        gn_stats_kernel<<<dim3(chunks, B), 256, 0, stream>>>(x, C, H, W, stats_ws);
    }
    MMDP_CUDA(cudaGetLastError());
    LaunchScope ls(LK_ROW, (double)B * npix * C * 8, stream);
    gn_apply_kernel<<<dim3(H + 2, B), 256, 0, stream>>>(x, y, C, H, W, stats_ws, gamma, beta, eps, swish, compact);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int upsample2x(const float* x, float* y, int B, int C, int H, int W, cudaStream_t stream) {
    if (C % 4) return set_error("upsample: channels must be a multiple of 4");
    LaunchScope ls(LK_ROW, (double)B * H * W * C * 4 * 5, stream);
    upsample2x_kernel<<<dim3(num_sms() * 8, B), 256, 0, stream>>>(x, y, C, H, W);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int softmax_rows_ld(float* s, int rows, int n, int ld, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)rows * n * 8, stream);
    softmax_rows_kernel<<<rows, 256, 0, stream>>>(s, n, ld);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// zero the one-pixel border of padded NHWC images
__global__ void zero_border_kernel(float* __restrict__ y, int C, int H, int W) {
    const int b = blockIdx.y, Wp = W + 2, Hp = H + 2;
    const int nb = 2 * Wp + 2 * H;  // border pixels per image
    const long long n = (long long)nb * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int j = (int)(i / C);
        int yy, xx;
        if (j < Wp) { yy = 0; xx = j; }
        else if (j < 2 * Wp) { yy = Hp - 1; xx = j - Wp; }
        else { const int r = j - 2 * Wp; yy = 1 + r / 2; xx = (r & 1) ? Wp - 1 : 0; }
        y[((size_t)b * Hp * Wp + (size_t)yy * Wp + xx) * C + c] = 0.f;
    }
}
int zero_border(float* y, int B, int C, int H, int W, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * (2 * (W + 2) + 2 * H) * C * 4, stream);
    zero_border_kernel<<<dim3(64, B), 256, 0, stream>>>(y, C, H, W);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int lfq_to_padded(const int64_t* ids, float* z, int B, int H, int W, int bits, int Cpad, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * H * W * (8 + 4.0 * bits), stream);
    lfq_to_padded_kernel<<<dim3((H * W + 255) / 256, B), 256, 0, stream>>>(ids, z, H, W, bits, Cpad);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int padded_to_nchw(const float* x, float* y, int B, int C, int ld, int H, int W, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * C * H * W * 8, stream);
    padded_to_nchw_kernel<<<dim3(num_sms() * 4, B), 256, 0, stream>>>(x, y, C, ld, H, W);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace mmdp
