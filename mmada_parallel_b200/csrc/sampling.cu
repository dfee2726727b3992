// The discrete-diffusion mask-predict step as HBM-bound kernels (warp-shuffle reductions, 16-byte loads):
//   text step  : MMaDA-Parallel-A/generators/parallel_generator.py:181-217  (M: models/modeling_mmada.py:179-209)
//   image step : MMaDA-Parallel-A/generators/parallel_generator.py:220-344  (M: models/modeling_mmada.py:211-241)
//   remask     : parallel_generator.py:23-70 mask_by_random_topk (A, exact-k from a stable ascending sort)
//                M/models/sampling.py:31-36 (M, strict '<' against the k-th smallest)
// All random numbers are INPUTS (drawn by the host from the same torch.Generator calls the reference makes), so the
// kernels are deterministic functions and can be checked bit-for-bit against the oracle.
// bf16 rounding points of the reference (python-scalar * bf16 tensor -> bf16, etc.) are reproduced explicitly.
#include "mmdp_internal.h"
#include "ptx.cuh"

#include <math.h>

namespace mmdp {

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x); f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z); f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}

// ------------------------------------------------------------------------------------------------
// text step, kernel 1: per-row argmax (first index on ties), fp64 softmax confidence of the argmax token
// ------------------------------------------------------------------------------------------------
struct TextRowArgs {
    const __nv_bfloat16* cond;    // [R, ld]
    const __nv_bfloat16* uncond;  // nullable; M: logits = cond + cfg * (uncond - cond), every op rounded to bf16
    const __nv_bfloat16* unoise;  // nullable; A gumbel: uniform noise [R, V] bf16 (torch.rand(dtype=bf16))
    const double* unoise64;       // nullable; M gumbel: uniform noise [R, V] fp64 (torch.rand_like(dtype=float64)), key =
                                  //   exp(logit) / (-log u)^temperature in fp64 (M/models/modeling_mmada.py:49-60)
    int64_t ld, ld_noise;
    int V;
    float cfg, temperature;
    int64_t* x0;    // [R]
    double* conf;   // [R]
};

__device__ __forceinline__ float text_logit(float c, float u, float cfg, bool has_uncond) {
    if (!has_uncond) return c;
    const float d = bf16_round(__fsub_rn(u, c));
    const float s = bf16_round(__fmul_rn(d, cfg));
    return bf16_round(__fadd_rn(c, s));
}
// logits + temperature * (-log(-log(u + 1e-10) + 1e-10)), all in bf16 (parallel_generator.py:8-20)
// g = -log(-log(u + eps) + eps), every op rounded to bf16 (eps = 1e-10: parallel_generator.py:8-20; 1e-20: utils/generation_utils.py:28-34)
__device__ __forceinline__ float gumbel_g_bf16(float u, float eps) {
    float t = bf16_round(__fadd_rn(u, eps));
    t = bf16_round(logf(t));
    t = -t;
    t = bf16_round(__fadd_rn(t, eps));
    t = bf16_round(logf(t));
    return -t;
}
__device__ __forceinline__ float gumbel_bf16(float logit, float u, float temperature) {
    const float t = bf16_round(__fmul_rn(gumbel_g_bf16(u, 1e-10f), temperature));
    return bf16_round(__fadd_rn(logit, t));
}

template <int kThreads>
__global__ void __launch_bounds__(kThreads) text_rows_kernel(TextRowArgs a) {
    const int row = blockIdx.x;
    const uint4* c4 = reinterpret_cast<const uint4*>(a.cond + (size_t)row * a.ld);
    const uint4* u4 = a.uncond ? reinterpret_cast<const uint4*>(a.uncond + (size_t)row * a.ld) : nullptr;
    const uint4* n4 = a.unoise ? reinterpret_cast<const uint4*>(a.unoise + (size_t)row * a.ld_noise) : nullptr;
    const int nvec = a.V / 8;
    const bool has_u = u4 != nullptr, has_n = n4 != nullptr;
    const double* n64 = a.unoise64 ? a.unoise64 + (size_t)row * a.ld_noise : nullptr;

    // pass 1: max of the (CFG-mixed) logits, argmax of the (optionally Gumbel-perturbed) logits
    float mx = -INFINITY;         // softmax max (un-noised)
    float best = -INFINITY;       // argmax key
    int best_i = 0x7fffffff;
    float best_logit = 0.f;       // un-noised logit at best_i
    if (n64) {
        // fp64 Gumbel-max of variant M: key = exp(double(l)) / (-log u)^T, first maximal index. The key is kept in fp64
        // (two floats would lose the tie behaviour); reduced across the CTA below through shared memory.
        double best_d = -INFINITY;
        const double T = (double)a.temperature;
        for (int i = threadIdx.x; i < nvec; i += kThreads) {
            float c[8], u[8];
            unpack8(c4[i], c);
            if (has_u) unpack8(u4[i], u);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float l = text_logit(c[j], has_u ? u[j] : 0.f, a.cfg, has_u);
                mx = fmaxf(mx, l);
                const double key = exp((double)l) / pow(-log(n64[(size_t)i * 8 + j]), T);
                if (key > best_d) { best_d = key; best_i = i * 8 + j; best_logit = l; }
            }
        }
        __shared__ double s_kd[kThreads / 32];
        __shared__ int s_ki[kThreads / 32];
        __shared__ float s_kl[kThreads / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best_d, o);
            const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
            const float ol = __shfl_xor_sync(0xffffffffu, best_logit, o);
            if (ob > best_d || (ob == best_d && oi < best_i)) { best_d = ob; best_i = oi; best_logit = ol; }
        }
        if ((threadIdx.x & 31) == 0) { s_kd[threadIdx.x >> 5] = best_d; s_ki[threadIdx.x >> 5] = best_i; s_kl[threadIdx.x >> 5] = best_logit; }
        __syncthreads();
        best_d = s_kd[0]; best_i = s_ki[0]; best_logit = s_kl[0];
        for (int i = 1; i < kThreads / 32; ++i)
            if (s_kd[i] > best_d || (s_kd[i] == best_d && s_ki[i] < best_i)) { best_d = s_kd[i]; best_i = s_ki[i]; best_logit = s_kl[i]; }
        __syncthreads();
        // hand the winner to the common reduction below as the only candidate of thread 0 (keys there are floats)
        best = threadIdx.x == 0 ? 1.0f : -INFINITY;
        if (threadIdx.x != 0) best_i = 0x7fffffff;
    } else
    for (int i0 = threadIdx.x; i0 < nvec; i0 += 4 * kThreads) {
        // four independent 16-byte loads per tensor in flight per thread (with one load at a time, one CTA of 16 warps per SM
        // leaves the kernel latency-bound)
        uint4 cv[4], uv[4], nv[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = i0 + t * kThreads;
            if (i < nvec) {
                cv[t] = c4[i];
                if (has_u) uv[t] = u4[i];
                if (has_n) nv[t] = n4[i];
            }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = i0 + t * kThreads;
            if (i >= nvec) break;
            float c[8], u[8], n[8];
            unpack8(cv[t], c);
            if (has_u) unpack8(uv[t], u);
            if (has_n) unpack8(nv[t], n);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float l = text_logit(c[j], has_u ? u[j] : 0.f, a.cfg, has_u);
                mx = fmaxf(mx, l);
                const float key = has_n ? gumbel_bf16(l, n[j], a.temperature) : l;
                if (key > best) { best = key; best_i = i * 8 + j; best_logit = l; }
            }
        }
    }
    __shared__ float s_f[kThreads / 32];
    __shared__ float s_best[kThreads / 32];
    __shared__ int s_idx[kThreads / 32];
    __shared__ float s_bl[kThreads / 32];
    __shared__ double s_d[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
        const float ol = __shfl_xor_sync(0xffffffffu, best_logit, o);
        if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; best_logit = ol; }
    }
    const int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
    if (ln == 0) { s_f[w] = mx; s_best[w] = best; s_idx[w] = best_i; s_bl[w] = best_logit; }
    __syncthreads();
    mx = s_f[0]; best = s_best[0]; best_i = s_idx[0]; best_logit = s_bl[0];
    for (int i = 1; i < kThreads / 32; ++i) {
        mx = fmaxf(mx, s_f[i]);
        if (s_best[i] > best || (s_best[i] == best && s_idx[i] < best_i)) { best = s_best[i]; best_i = s_idx[i]; best_logit = s_bl[i]; }
    }

    // pass 2 (row now L2-resident): sum exp(l - max) in fp64 == F.softmax(logits.to(float64)) denominator.
    // A bf16 logit takes few distinct values: exp(double(v) - max) is tabulated once per row for every bf16 pattern with
    // 2^-6 <= |v| < 2^6 (2 signs x 12 exponents x 128 mantissas = 24 KB of shared memory, 6 fp64 exp per thread) and the pass
    // becomes a table gather + fp64 add - the ~0.5 % of the elements outside the window take the direct exp. The terms are
    // bit-identical to the direct evaluation (same expression), only their summation order is the kernel's own.
    constexpr int kTabExp0 = 121, kTabExps = 12;                 // biased bf16 exponents [121, 133)
    __shared__ double s_tab[2 * kTabExps * 128];
    const double dmx = (double)mx;
    for (int t = threadIdx.x; t < 2 * kTabExps * 128; t += kThreads) {
        const uint32_t sgn = t / (kTabExps * 128), rem = t - sgn * (kTabExps * 128);
        const uint32_t bits = (sgn << 15) | ((kTabExp0 + rem / 128) << 7) | (rem & 127);
        const double d = (double)__uint_as_float(bits << 16) - dmx;
        s_tab[t] = d > -64.0 ? exp(d) : 0.0;                    // exp(-64) < 2^-92: below half an ulp of any fp64 sum >= 1
    }
    __syncthreads();
    double sum = 0.0;
    for (int i0 = threadIdx.x; i0 < nvec; i0 += 4 * kThreads) {
        uint4 cv[4], uv[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = i0 + t * kThreads;
            if (i < nvec) {
                cv[t] = c4[i];
                if (has_u) uv[t] = u4[i];
            }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int i = i0 + t * kThreads;
            if (i >= nvec) break;
            float c[8], u[8];
            unpack8(cv[t], c);
            if (has_u) unpack8(uv[t], u);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float l = text_logit(c[j], has_u ? u[j] : 0.f, a.cfg, has_u);
                const uint32_t b = __float_as_uint(l) >> 16;
                const uint32_t e = ((b >> 7) & 0xffu) - kTabExp0;
                if (e < (uint32_t)kTabExps) {
                    sum += s_tab[((b >> 15) * kTabExps + e) * 128 + (b & 127u)];
                } else {
                    const double d = (double)l - dmx;
                    if (d > -64.0) sum += exp(d);
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (ln == 0) s_d[w] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int i = 0; i < kThreads / 32; ++i) tot += s_d[i];
        a.x0[row] = best_i;
        a.conf[row] = exp((double)best_logit - dmx) / tot;
    }
}

// text step, kernel 2: confidence top-k (k largest, ties -> lower index) and commit into the id buffer
static constexpr int kTextMaxR = 4096;
__global__ void __launch_bounds__(1024) text_commit_kernel(const int64_t* __restrict__ x0, const double* __restrict__ conf, int64_t* ids, int R,
                                                           int64_t mask_id, int k) {
    extern __shared__ double s_confd[];
    for (int i = threadIdx.x; i < R; i += blockDim.x) s_confd[i] = (ids[i] == mask_id) ? conf[i] : -INFINITY;
    __syncthreads();
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
        const bool masked = ids[i] == mask_id;  // (only this thread writes ids[i])
        const double c = s_confd[i];
        int rank = 0;
        for (int j = 0; j < R; ++j) {
            const double cj = s_confd[j];
            rank += (cj > c) || (cj == c && j < i);
        }
        if (rank < k && masked) ids[i] = x0[i];
    }
}

int text_step(const __nv_bfloat16* cond, const __nv_bfloat16* uncond, int64_t ld, int R, int V, float text_cfg,
              const __nv_bfloat16* unoise, int64_t ld_noise, float temperature, int64_t* ids_text, int64_t mask_id,
              int k, int64_t* x0_ws, double* conf_ws, cudaStream_t stream, const double* unoise64) {
    if (R <= 0) return 0;
    if (unoise && unoise64) return set_error("text_step: bf16 and fp64 Gumbel noise are mutually exclusive");
    if (R > kTextMaxR) return set_error("text_step: at most %d text positions", kTextMaxR);
    if ((V % 8) || (ld % 8) || (unoise && (ld_noise % 8))) return set_error("text_step: V/ld must be multiples of 8");
    TextRowArgs a{cond, uncond, unoise, unoise64, ld, ld_noise, V, text_cfg, temperature, x0_ws, conf_ws};
    {
        LaunchScope ls(LK_SAMPLE, (double)R * V * 2 * (uncond ? 2 : 1) + (unoise ? (double)R * V * 2 : 0) + (unoise64 ? (double)R * V * 8 : 0), stream);  // bytes read
        text_rows_kernel<512><<<R, 512, 0, stream>>>(a);
    }
    MMDP_CUDA(cudaGetLastError());
    const int threads = R >= 1024 ? 1024 : ((R + 31) / 32) * 32;
    LaunchScope ls2(LK_SAMPLE, (double)R * 24, stream);
    text_commit_kernel<<<1, threads, R * sizeof(double), stream>>>(x0_ws, conf_ws, ids_text, R, mask_id, k);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// image step, kernel 1: per VQ position: CFG mix -> softmax (bf16 probs) -> argmax | exponential-race sample
// ------------------------------------------------------------------------------------------------
struct ImageRowArgs {
    const __nv_bfloat16* cond;   // row r at cond + r*ld, `C` codebook logits
    const __nv_bfloat16* unc_a;  // A: uncond_text (scale s_a) | M: uncond (scale s_a = image_cfg)
    const __nv_bfloat16* unc_b;  // A: uncond_image (scale s_b) | M: unused
    int64_t ld;
    int C;           // codebook size (multiple of 8, <= 8192)
    int variant;     // 0 = A, 1 = M
    float s_a, s_b;
    const __nv_bfloat16* qnoise;  // nullable: Exp(1) noise [N, C] bf16 (torch.multinomial's q); null -> argmax(probs)
    const __nv_bfloat16* gumbel_u;  // nullable: uniform noise [N, C] bf16 -> Gumbel-max on the LOGITS, argmax(l / tau + g)
    float gumbel_tau;               //   (A/utils/generation_utils.py:37-42); sample_logits != 0 with gumbel_u null = argmax(l)
    int sample_logits;              // 0: sample from the bf16 probabilities (argmax | exponential race); 1: from the logits
    const int64_t* ids;           // full id buffer
    const int* pos;               // [N] sequence position of VQ token r
    int64_t mask_id, vq_offset;
    int clamp_known;              // A clamps known ids into [0, C-1]; M does not
    int32_t* sampled;             // [N] out: where(unknown, sample, known)
    float* selp;                  // [N] out: prob of the chosen id as bf16 value (or bf16 finfo.max for known)
    uint8_t* unknown;             // [N] out
    __nv_bfloat16* probs_out;     // nullable debug: [N, C]
};

static constexpr int kImgThreads = 256;
static constexpr int kImgMaxPer = 4;  // 256 threads * 4 vec8 = 8192 columns

__global__ void __launch_bounds__(kImgThreads) image_rows_kernel(ImageRowArgs a) {
    const int r = blockIdx.x;
    const int nvec = a.C / 8;
    const uint4* c4 = reinterpret_cast<const uint4*>(a.cond + (size_t)r * a.ld);
    const uint4* ua4 = a.unc_a ? reinterpret_cast<const uint4*>(a.unc_a + (size_t)r * a.ld) : nullptr;
    const uint4* ub4 = a.unc_b ? reinterpret_cast<const uint4*>(a.unc_b + (size_t)r * a.ld) : nullptr;

    float x[kImgMaxPer][8];
    float mx = -INFINITY;
    // logits-domain sampling (generate_image): the key is formed here, where the mixed logit is at hand
    const uint4* g4 = a.gumbel_u ? reinterpret_cast<const uint4*>(a.gumbel_u + (size_t)r * a.C) : nullptr;
    float lbest = -INFINITY;
    int lbest_i = 0x7fffffff;
#pragma unroll
    for (int t = 0; t < kImgMaxPer; ++t) {
        const int i = threadIdx.x + t * kImgThreads;
        if (i < nvec) {
            float c[8], ua[8], ub[8], gu[8];
            unpack8(c4[i], c);
            if (ua4) unpack8(ua4[i], ua);
            if (ub4) unpack8(ub4[i], ub);
            if (g4) unpack8(g4[i], gu);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float l = c[j];
                if (a.variant == 0) {
                    // image_logits = cond; += s_t * (cond - unc_t); += s_i * (cond - unc_i)   (bf16 at every op)
                    if (ua4 && a.s_a != 0.f) l = bf16_round(__fadd_rn(l, bf16_round(__fmul_rn(bf16_round(__fsub_rn(c[j], ua[j])), a.s_a))));
                    if (ub4 && a.s_b != 0.f) l = bf16_round(__fadd_rn(l, bf16_round(__fmul_rn(bf16_round(__fsub_rn(c[j], ub[j])), a.s_b))));
                } else {
                    // (1 + s) * cond - s * uncond   (s_b carries the host-evaluated python float 1 + s)
                    const float p1 = bf16_round(__fmul_rn(c[j], a.s_b));
                    const float p2 = bf16_round(__fmul_rn(ua[j], a.s_a));
                    l = bf16_round(__fsub_rn(p1, p2));
                }
                x[t][j] = l;
                mx = fmaxf(mx, l);
                if (a.sample_logits) {
                    // (logits / tau + g).argmax(): bf16 at every op; tau == 0 is the plain argmax of the logits
                    const float key = g4 ? bf16_round(__fadd_rn(bf16_round(__fdiv_rn(l, a.gumbel_tau)), gumbel_g_bf16(gu[j], 1e-20f))) : l;
                    if (key > lbest) { lbest = key; lbest_i = i * 8 + j; }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) x[t][j] = -INFINITY;
        }
    }
    __shared__ float s_f[kImgThreads / 32];
    __shared__ int s_i[kImgThreads / 32];
    __shared__ float s_p[kImgThreads / 32];
    const int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (ln == 0) s_f[w] = mx;
    __syncthreads();
    mx = s_f[0];
    for (int i = 1; i < kImgThreads / 32; ++i) mx = fmaxf(mx, s_f[i]);
    __syncthreads();

    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < kImgMaxPer; ++t)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e = expf(__fsub_rn(x[t][j], mx));
            x[t][j] = e;
            sum += e;
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (ln == 0) s_f[w] = sum;
    __syncthreads();
    sum = 0.f;
    for (int i = 0; i < kImgThreads / 32; ++i) sum += s_f[i];

    // probs (bf16), then the sampling key: argmax(probs) or argmax(bf16(probs / q))
    const int64_t tok = a.ids[a.pos[r]];
    const bool unk = tok == a.mask_id;
    const uint4* q4 = a.qnoise ? reinterpret_cast<const uint4*>(a.qnoise + (size_t)r * a.C) : nullptr;
    float best = -INFINITY, best_p = 0.f;
    int best_i = 0x7fffffff;
    int64_t known = tok - a.vq_offset;
    if (a.clamp_known) known = known < 0 ? 0 : (known > a.C - 1 ? a.C - 1 : known);
#pragma unroll
    for (int t = 0; t < kImgMaxPer; ++t) {
        const int i = threadIdx.x + t * kImgThreads;
        if (i < nvec) {
            float q[8];
            if (q4) unpack8(q4[i], q);
            uint32_t pk[4];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float p = bf16_round(__fdiv_rn(x[t][j], sum));
                x[t][j] = p;
                if (a.sample_logits) {
                    if (i * 8 + j == lbest_i) { best = lbest; best_i = lbest_i; best_p = p; }
                } else {
                    const float key = q4 ? bf16_round(__fdiv_rn(p, q[j])) : p;
                    if (key > best) { best = key; best_i = i * 8 + j; best_p = p; }
                }
            }
            if (a.probs_out) {
#pragma unroll
                for (int j = 0; j < 4; ++j) pk[j] = pack_bf16x2(x[t][2 * j], x[t][2 * j + 1]);
                reinterpret_cast<uint4*>(a.probs_out + (size_t)r * a.C)[i] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
        const float op = __shfl_xor_sync(0xffffffffu, best_p, o);
        if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; best_p = op; }
    }
    if (ln == 0) { s_f[w] = best; s_i[w] = best_i; s_p[w] = best_p; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < kImgThreads / 32; ++i)
            if (s_f[i] > best || (s_f[i] == best && s_i[i] < best_i)) { best = s_f[i]; best_i = s_i[i]; best_p = s_p[i]; }
        int samp = best_i;
        if (samp > a.C - 1) samp = a.C - 1;  // also covers the (all-NaN) nothing-selected case
        a.unknown[r] = unk ? 1 : 0;
        if (unk) {
            a.sampled[r] = samp;
            a.selp[r] = best_p;
        } else {
            a.sampled[r] = (int32_t)known;
            a.selp[r] = 3.3895313892515355e38f;  // torch.finfo(torch.bfloat16).max
        }
    }
}

// ------------------------------------------------------------------------------------------------
// image step, kernel 2 (single CTA): confidence jitter -> stable rank -> re-mask -> write ids
// ------------------------------------------------------------------------------------------------
struct RemaskArgs {
    int N;                 // number of VQ tokens (<= kRemaskMaxN)
    int variant;           // 0 = A, 1 = M
    const int32_t* sampled;
    const float* selp;
    const uint8_t* unknown;
    const __nv_bfloat16* noise;  // A: randn [N] bf16 ; M: uniform [N] bf16 ; nullable when temp == 0
    float temp;                  // temperature * (1 - ratio)
    int sched_len;               // floor(N * noise_schedule(ratio)) evaluated on the host exactly as the reference does
    int64_t* ids;
    const int* pos;
    int64_t mask_id, vq_offset;
    int32_t* mask_len_out;       // nullable debug
    uint8_t* masking_out;        // nullable debug [N]
    int k_direct;                // >= 0: the number of the cut-off element is given (clamped to [0, N-1]) instead of the
                                 //   max(1, min(unknown - 1, sched_len)) rule (generate_image passes keep_n, :99-103)
};

__device__ __forceinline__ float log_bf16(float x) { return bf16_round(logf(x)); }

static constexpr int kRemaskMaxN = 4096;  // 768x768 images of the reference app are 2304 VQ tokens
static constexpr int kRemaskPer = kRemaskMaxN / 1024;

__global__ void __launch_bounds__(1024) image_remask_kernel(RemaskArgs a) {
    extern __shared__ float s_conf[];  // [N]
    __shared__ int s_cnt[32];
    __shared__ float s_cut;
    const int tid = threadIdx.x;
    int cnt = 0;
    float conf[kRemaskPer];
#pragma unroll
    for (int t = 0; t < kRemaskPer; ++t) {
        const int i = tid + t * 1024;
        conf[t] = INFINITY;
        if (i >= a.N) continue;
        cnt += a.unknown[i] ? 1 : 0;
        const float p = a.selp[i];
        const float nz = a.noise ? __bfloat162float(a.noise[i]) : 0.f;
        if (a.variant == 0) {
            // confidence = log(probs + 1e-10) + temperature * noise     (parallel_generator.py:36)
            const float lp = log_bf16(bf16_round(__fadd_rn(p, 1e-10f)));
            const float tn = a.noise ? bf16_round(__fmul_rn(nz, a.temp)) : 0.f;
            conf[t] = bf16_round(__fadd_rn(lp, tn));
        } else if (a.variant == 1) {
            // confidence = log(clamp(p,1e-20)) + temperature * (-log(clamp(-log(clamp(u,1e-20)),1e-20)))  (sampling.py:9-16,31-32)
            const float lp = log_bf16(fmaxf(p, bf16_round(1e-20f)));
            float g = 0.f;
            if (a.noise) {
                g = log_bf16(fmaxf(nz, bf16_round(1e-20f)));
                g = -g;
                g = log_bf16(fmaxf(g, bf16_round(1e-20f)));
                g = -g;
            }
            const float tn = bf16_round(__fmul_rn(g, a.temp));
            conf[t] = bf16_round(__fadd_rn(lp, tn));
        } else {
            // variant 2 (A/utils/generation_utils.py:45-61): log(clamp_min(p,1e-20)) + temperature * (-log(-log(u+1e-20)+1e-20))
            const float lp = log_bf16(fmaxf(p, bf16_round(1e-20f)));
            const float g = a.noise ? gumbel_g_bf16(nz, 1e-20f) : 0.f;
            const float tn = bf16_round(__fmul_rn(g, a.temp));
            conf[t] = bf16_round(__fadd_rn(lp, tn));
        }
        s_conf[i] = conf[t];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((tid & 31) == 0) s_cnt[tid >> 5] = cnt;
    __syncthreads();
    int unknown_cnt = 0;
    for (int j = 0; j < 32; ++j) unknown_cnt += s_cnt[j];
    // mask_len = max(1, min(unknown - 1, sched_len))
    int k = a.sched_len < unknown_cnt - 1 ? a.sched_len : unknown_cnt - 1;
    if (k < 1) k = 1;
    if (a.k_direct >= 0) k = a.k_direct;
    if (a.variant == 0 || a.k_direct >= 0) { if (k > a.N - 1) k = a.N - 1; if (k < 0) k = 0; }  // mask_by_random_topk clamps to [0, N-1]
    int rank[kRemaskPer];
#pragma unroll
    for (int t = 0; t < kRemaskPer; ++t) {
        const int i = tid + t * 1024;
        rank[t] = 0;
        if (i >= a.N) continue;
        const float c = conf[t];
        int r = 0;
        for (int j = 0; j < a.N; ++j) {
            const float cj = s_conf[j];
            r += (cj < c) || (cj == c && j < i);  // stable ascending sort position
        }
        rank[t] = r;
        if (a.variant != 0 && r == (k < a.N ? k : a.N - 1)) s_cut = c;  // sorted_confidence[mask_len]
    }
    if (a.variant != 0) __syncthreads();
#pragma unroll
    for (int t = 0; t < kRemaskPer; ++t) {
        const int i = tid + t * 1024;
        if (i >= a.N) continue;
        const bool masking = a.variant == 0 ? rank[t] < k : conf[t] < s_cut;
        a.ids[a.pos[i]] = masking ? a.mask_id : (int64_t)a.sampled[i] + a.vq_offset;
        if (a.masking_out) a.masking_out[i] = masking ? 1 : 0;
    }
    if (tid == 0 && a.mask_len_out) *a.mask_len_out = k;
}

int image_remask(int variant, int N, const int32_t* sampled, const float* selp, const uint8_t* unknown,
                 const __nv_bfloat16* conf_noise, float temp, int sched_len, int64_t* ids, const int* pos, int64_t mask_id,
                 int64_t vq_offset, int32_t* mask_len_out, uint8_t* masking_out, cudaStream_t stream, int k_direct) {
    if (N <= 0 || N > kRemaskMaxN) return set_error("image_remask: N must be in [1, %d]", kRemaskMaxN);
    RemaskArgs ma{N, variant, sampled, selp, unknown, conf_noise, temp, sched_len, ids, pos, mask_id, vq_offset,
                  mask_len_out, masking_out, k_direct};
    LaunchScope ls(LK_SAMPLE, (double)N * 24, stream);
    image_remask_kernel<<<1, 1024, N * sizeof(float), stream>>>(ma);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

int image_step(int variant, const __nv_bfloat16* cond, const __nv_bfloat16* unc_a, const __nv_bfloat16* unc_b, int64_t ld,
               int N, int C, float s_a, float s_b, const __nv_bfloat16* qnoise, const __nv_bfloat16* conf_noise,
               float temp, int sched_len, int64_t* ids, const int* pos, int64_t mask_id, int64_t vq_offset,
               int32_t* sampled_ws, float* selp_ws, uint8_t* unknown_ws, __nv_bfloat16* probs_out,
               int32_t* mask_len_out, uint8_t* masking_out, cudaStream_t stream) {
    if (N <= 0 || N > kRemaskMaxN) return set_error("image_step: N must be in [1, %d]", kRemaskMaxN);
    if (C <= 0 || (C % 8) || C > kImgThreads * kImgMaxPer * 8) return set_error("image_step: codebook size must be a multiple of 8 and <= 8192");
    if (ld % 8) return set_error("image_step: ld must be a multiple of 8");
    if (variant == 1 && !unc_a) return set_error("image_step: variant M needs uncond logits");
    ImageRowArgs ra{cond, unc_a, unc_b, ld, C, variant, s_a, s_b, qnoise, nullptr, 0.f, 0, ids, pos, mask_id, vq_offset,
                    variant == 0 ? 1 : 0, sampled_ws, selp_ws, unknown_ws, probs_out};
    {
        const int nt = 1 + (unc_a ? 1 : 0) + (unc_b ? 1 : 0) + (qnoise ? 1 : 0);
        LaunchScope ls(LK_SAMPLE, (double)N * C * 2 * nt, stream);  // bytes read
        image_rows_kernel<<<N, kImgThreads, 0, stream>>>(ra);
    }
    MMDP_CUDA(cudaGetLastError());
    return image_remask(variant, N, sampled_ws, selp_ws, unknown_ws, conf_noise, temp, sched_len, ids, pos, mask_id,
                        vq_offset, mask_len_out, masking_out, stream);
}

// One step of A's MaskGit text-to-image decoding (generators/image_generation_generator.py:119-208) on the N currently
// masked positions `pos` (compacted by the caller): logits = cond | (1 + s) cond - s uncond, Gumbel-max sample on the logits
// (utils/generation_utils.py:37-42), confidence = softmax probability of the sample, write-back, then re-mask every
// position whose noisy log-confidence is below the keep_n-th smallest (generation_utils.py:45-61).
int image_step_t2i(const __nv_bfloat16* cond, const __nv_bfloat16* uncond, int64_t ld, int N, int C, float cfg,
                   const __nv_bfloat16* gumbel_u, float tau, const __nv_bfloat16* conf_u, float temperature, int keep_n,
                   int64_t* ids, const int* pos, int64_t mask_id, int64_t vq_offset, int32_t* sampled_ws, float* selp_ws,
                   uint8_t* unknown_ws, uint8_t* masking_out, cudaStream_t stream) {
    if (N <= 0 || N > kRemaskMaxN) return set_error("image_step_t2i: N must be in [1, %d]", kRemaskMaxN);
    if (C <= 0 || (C % 8) || C > kImgThreads * kImgMaxPer * 8) return set_error("image_step_t2i: codebook size must be a multiple of 8 and <= 8192");
    if (ld % 8) return set_error("image_step_t2i: ld must be a multiple of 8");
    if (gumbel_u && tau == 0.f) return set_error("image_step_t2i: Gumbel noise given with tau == 0");
    // CFG mix = variant M's formula with s_a = s (python float), s_b = 1 + s evaluated on the host in double like the reference
    ImageRowArgs ra{cond, uncond, nullptr, ld, C, uncond ? 1 : 0, cfg, (float)(1.0 + (double)cfg), nullptr, gumbel_u, tau, 1, ids, pos,
                    mask_id, vq_offset, 0, sampled_ws, selp_ws, unknown_ws, nullptr};
    {
        LaunchScope ls(LK_SAMPLE, (double)N * C * 2 * (1 + (uncond ? 1 : 0) + (gumbel_u ? 1 : 0)), stream);
        image_rows_kernel<<<N, kImgThreads, 0, stream>>>(ra);
    }
    MMDP_CUDA(cudaGetLastError());
    return image_remask(2, N, sampled_ws, selp_ws, unknown_ws, conf_u, temperature, 0, ids, pos, mask_id, vq_offset, nullptr,
                        masking_out, stream, keep_n < 0 ? 0 : keep_n);
}

}  // namespace mmdp
