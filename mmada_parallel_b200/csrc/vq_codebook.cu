// Learned-codebook kernels of the aMUSEd VQ-VAE (diffusers VectorQuantizer, autoencoders/vae.py):
//   codebook_to_padded  get_codebook_entry: ids [B, h*w] -> rows of the codebook, written straight into the padded
//                       channels-last input of the decoder (the layout of conv_tf32.cu)
//   vq_nearest          forward's argmin: for every latent vector z the index of the code e minimising sum_c (z_c - e_c)^2,
//                       lowest index on ties. Exact fp32 SIMT arithmetic, not TF32: at 64 channels TF32 products move a
//                       distance by ~1e-3 relative, enough to swap close winners, and the work (1 GFLOP for 1024 latents x
//                       8192 codes) is too small to need tensor cores. Codebook tiles live in shared memory and the argmin is
//                       fused: no [N, n_codes] distance matrix is written.
#include "../../include/mmdp.h"
#include "mmdp_internal.h"

namespace mmdp {

// ---- gather -------------------------------------------------------------------------------------------------------
// z [B, (h+2)(w+2), Cpad]: interior pixel (y, x) of image b gets codebook row ids[b, y*w + x]; channels >= C and the border
// are left as they are (the caller zeroes the buffer). An id outside [0, n_codes) raises bit 0 of *err and writes zeros.
__global__ void __launch_bounds__(256) codebook_to_padded_kernel(const int64_t* __restrict__ ids, const float* __restrict__ cb,
                                                                 float* __restrict__ z, int h, int w, int C, int Cpad,
                                                                 int64_t n_codes, int* __restrict__ err) {
    const int b = blockIdx.y;
    const long long n = (long long)h * w * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int p = (int)(i / C);
        const int64_t id = ids[(size_t)b * h * w + p];
        float v = 0.f;
        if (id >= 0 && id < n_codes)
            v = cb[(size_t)id * C + c];
        else if (c == 0)
            atomicOr(err, 1);
        const int y = p / w, x = p - y * w;
        z[((size_t)b * (h + 2) * (w + 2) + (size_t)(y + 1) * (w + 2) + x + 1) * Cpad + c] = v;
    }
}

int codebook_to_padded(const int64_t* ids, const float* cb, float* z, int B, int h, int w, int C, int Cpad, int64_t n_codes,
                       int* err, cudaStream_t stream) {
    LaunchScope ls(LK_ROW, (double)B * h * w * (8 + 8.0 * C), stream);
    codebook_to_padded_kernel<<<dim3(num_sms() * 2, B), 256, 0, stream>>>(ids, cb, z, h, w, C, Cpad, n_codes, err);
    MMDP_CUDA(cudaGetLastError());
    return 0;
}

// ---- nearest code -------------------------------------------------------------------------------------------------
// CTA = 32 latent vectors x a contiguous range of codes, 256 threads. Thread (tv, tc) owns vectors 2tv, 2tv+1 and, per tile
// of 64 codes, codes tc, tc+16, tc+32, tc+48: eight running sums of (z_c - e_c)^2 over c = 0..C-1 in order (fmaf), so a
// distance does not depend on the launch shape. Each thread keeps the first minimum over its codes (increasing index), the 16
// threads of a vector reduce (distance, index) lexicographically, and one atomicMin per vector and CTA merges the code
// ranges: distances are >= 0, so their fp32 bit patterns order like the values, and (bits << 32 | index) keeps the lowest
// index on a tie. The packed minimum lives in ids_out itself and is unpacked in place afterwards.
static constexpr int kNnVec = 32, kNnCodes = 64, kNnThreads = 256;

__global__ void __launch_bounds__(kNnThreads) vq_nearest_kernel(const float* __restrict__ z, const float* __restrict__ cb, int C,
                                                                int hw, int N, int n_codes, int codes_per_cta,
                                                                unsigned long long* __restrict__ best) {
    extern __shared__ float nn_smem[];
    float* zs = nn_smem;                 // [C][kNnVec]
    float* es = nn_smem + C * kNnVec;    // [kNnCodes][C + 1] (odd row stride: the 16 code lanes hit 16 banks)
    const int ld = C + 1;
    const int v0 = blockIdx.x * kNnVec;
    for (int i = threadIdx.x; i < C * kNnVec; i += kNnThreads) {
        const int c = i / kNnVec, v = i - c * kNnVec, n = v0 + v;
        float val = 0.f;
        if (n < N) {
            const int b = n / hw, p = n - b * hw;
            val = z[((size_t)b * C + c) * hw + p];
        }
        zs[i] = val;
    }
    const int tv = threadIdx.x >> 4, tc = threadIdx.x & 15;
    float bd[2] = {INFINITY, INFINITY};
    int bi[2] = {0x7fffffff, 0x7fffffff};
    const int c_begin = blockIdx.y * codes_per_cta;
    const int c_end = min(n_codes, c_begin + codes_per_cta);
    for (int t0 = c_begin; t0 < c_end; t0 += kNnCodes) {
        __syncthreads();  // the previous tile is consumed (first pass: the z tile is written)
        for (int i = threadIdx.x; i < C * kNnCodes; i += kNnThreads) {
            const int j = i / C, c = i - j * C;
            es[j * ld + c] = t0 + j < c_end ? cb[(size_t)(t0 + j) * C + c] : 0.f;
        }
        __syncthreads();
        float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll 4
        for (int c = 0; c < C; ++c) {
            const float2 zv = *reinterpret_cast<const float2*>(&zs[c * kNnVec + 2 * tv]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float e = es[(tc + 16 * k) * ld + c];
                const float d0 = zv.x - e, d1 = zv.y - e;
                acc[0][k] = fmaf(d0, d0, acc[0][k]);
                acc[1][k] = fmaf(d1, d1, acc[1][k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int code = t0 + tc + 16 * k;
            if (code < c_end) {
#pragma unroll
                for (int v = 0; v < 2; ++v)
                    if (acc[v][k] < bd[v] || bi[v] == 0x7fffffff) { bd[v] = acc[v][k]; bi[v] = code; }
            }
        }
    }
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        float d = bd[v];
        int idx = bi[v];
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(0xffffffffu, d, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (od < d || (od == d && oi < idx)) { d = od; idx = oi; }
        }
        const int n = v0 + 2 * tv + v;
        if (tc == 0 && n < N)
            atomicMin(&best[n], ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)idx);
    }
}

// ids[n] = low 32 bits of the packed minimum (in place)
__global__ void vq_unpack_kernel(int64_t* __restrict__ ids, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < N) ids[n] = (int64_t)(reinterpret_cast<unsigned long long*>(ids)[n] & 0xffffffffull);
}

// z_q [B, C, h, w] = codebook rows of ids [B, h*w]
__global__ void __launch_bounds__(256) vq_gather_nchw_kernel(const int64_t* __restrict__ ids, const float* __restrict__ cb,
                                                             float* __restrict__ zq, int C, int hw, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(i % hw);
        const long long bc = i / hw;
        const int c = (int)(bc % C), b = (int)(bc / C);
        zq[i] = cb[(size_t)ids[(size_t)b * hw + p] * C + c];
    }
}

int vq_nearest(const float* z, const float* cb, int B, int C, int h, int w, int n_codes, int64_t* ids, float* zq,
               cudaStream_t stream) {
    if (B < 1 || C < 1 || C > 256 || h < 1 || w < 1 || n_codes < 1)
        return set_error("vq_nearest: bad shape (B=%d C=%d h=%d w=%d n_codes=%d; C must be in [1, 256])", B, C, h, w, n_codes);
    const long long Nl = (long long)B * h * w;
    if (Nl > 0x7fffffffLL) return set_error("vq_nearest: too many latent vectors");
    const int N = (int)Nl, hw = h * w;
    const int smem = (C * kNnVec + kNnCodes * (C + 1)) * 4;
    static unsigned long long attr_set = 0;  // bit per device: the attribute is a property of each device's module
    int dev = 0;
    MMDP_CUDA(cudaGetDevice(&dev));
    if (!(attr_set >> (dev & 63) & 1ull)) {
        MMDP_CUDA(cudaFuncSetAttribute(vq_nearest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (256 * kNnVec + kNnCodes * 257) * 4));
        attr_set |= 1ull << (dev & 63);
    }
    // split the codebook so that about two CTAs per SM run
    const int gx = (N + kNnVec - 1) / kNnVec;
    const int tiles = (n_codes + kNnCodes - 1) / kNnCodes;
    int splits = (2 * num_sms() + gx - 1) / gx;
    if (splits > tiles) splits = tiles;
    if (splits < 1) splits = 1;
    const int per = (tiles + splits - 1) / splits * kNnCodes;
    splits = (n_codes + per - 1) / per;
    MMDP_CUDA(cudaMemsetAsync(ids, 0xff, (size_t)N * 8, stream));
    {
        LaunchScope ls(LK_ROW, (double)n_codes * C * 4 * gx + (double)N * C * 4, stream);
        vq_nearest_kernel<<<dim3(gx, splits), kNnThreads, smem, stream>>>(z, cb, C, hw, N, n_codes, per,
                                                                          reinterpret_cast<unsigned long long*>(ids));
        MMDP_CUDA(cudaGetLastError());
    }
    {
        LaunchScope ls(LK_ROW, (double)N * 16, stream);
        vq_unpack_kernel<<<(N + 255) / 256, 256, 0, stream>>>(ids, N);
        MMDP_CUDA(cudaGetLastError());
    }
    if (zq) {
        const long long total = (long long)N * C;
        LaunchScope ls(LK_ROW, (double)total * 8, stream);
        vq_gather_nchw_kernel<<<num_sms() * 4, 256, 0, stream>>>(ids, cb, zq, C, hw, total);
        MMDP_CUDA(cudaGetLastError());
    }
    return 0;
}

}  // namespace mmdp

extern "C" MMDP_API int mmdp_vq_nearest(const float* latents_nchw, const float* codebook, int B, int C, int h, int w, int n_codes,
                                        int64_t* ids_out, float* zq_nchw, void* stream) {
    if (!latents_nchw || !codebook || !ids_out) return mmdp::set_error("mmdp_vq_nearest: null argument");
    return mmdp::vq_nearest(latents_nchw, codebook, B, C, h, w, n_codes, ids_out, zq_nchw, (cudaStream_t)stream);
}
