// Tensor-parallel collective of the single-sample forward (BASELINE config 4), written against NVLink peer memory instead of
// NCCL. Rank r owns the rows [r*R, (r+1)*R) of the residual stream (R = ceil(M / TP)). The two row-parallel GEMMs of a
// layer (attn_out, ff_out; modeling_llada.py:744, :968) PUSH their fp32 partial rows from the epilogue straight into the
// owner's receive buffer over NVLink (gemm_epilogue.cuh, EPI_F32 scatter: the reduce-scatter is fused into the GEMM and
// overlaps its main loop; pulls over NVLink measured 2-3x slower than pushes). What follows in the reference - residual add
// (:953 / :970), the next RMSLayerNorm (:315-329) and the broadcast of its output to all ranks - is ONE kernel per rank:
//
//     sum   = part_0[row] + part_1[row] + ... + part_{TP-1}[row]      fp32, fixed rank order (local loads of the pushed rows)
//     x     = bf16( bf16(sum) + x )                                   the single-GPU rounding points of EPI_RESID
//     xn    = bf16( w * bf16( x * rsqrt(mean(x^2) + eps) ) )          RMSLayerNorm with the next norm's weight
//     xn -> every rank's activation buffer                            P2P stores over NVLink (the all-gather)
//
// i.e. reduce-scatter(fp32) + residual + norm + all-gather(bf16): 0.75x the bytes of the fp32 all-reduce it replaces, no
// separate residual / RMSNorm launches, and the summation order is the same on every rank and in every run.
// Synchronisation is a flag per (phase, source rank) in each rank's memory, written by the peers with system-scope
// release stores: phase 0 "my partial sums are complete" (sent by tp_rendezvous_kernel, a one-CTA launch that follows the
// producing GEMM in stream order and waits for everybody's), phase 1 "my rows of xn have landed in your buffer" (sent by the last CTA). The consumer of xn waits for
// phase 1 of all ranks in tp_wait_kernel. Flags carry a monotonically increasing epoch, so they never need resetting.
// Buffer reuse is safe with TWO partial buffers used alternately (a rank can only overwrite a partial buffer two
// collectives later, after it has itself passed the next phase-0 barrier, which every peer joins only after its reads).
//
// FP8 form (tp_reduce_norm_fp8, the tensor-parallel forward with e4m3 block linears): the normalised bf16 row is not stored
// but quantised on the spot, exactly as quantize_fp8 (fp8.cu, group 128) would quantise it - a 128-column group is the 16
// consecutive threads of a half-warp, amax by half-warp shuffles, s = amax / 448 (1 for an all-zero group), q = e4m3(x / s) -
// and the e4m3 bytes plus the group scales go to every rank: d + d/32 bytes per row instead of 2d, and no rank has to
// quantise the replicated activations itself before its next column-parallel GEMM.
#include "mmdp_internal.h"
#include "ptx.cuh"

namespace mmdp {

static constexpr int kTpMaxRanks = 8;
static constexpr int kTpThreads = 256;

struct TpReduceArgs {
    const float* part[kTpMaxRanks];      // partial sums of every rank FOR THIS RANK'S ROWS: slot r of the local receive buffer,
                                         // [rows_per_rank, d] fp32, pushed there by rank r's GEMM epilogue (unused when n_src == 0)
    __nv_bfloat16* xn[kTpMaxRanks];      // activation buffer of every rank, peer-mapped; [M, d] bf16
    uint32_t* flags[kTpMaxRanks];        // flag array of every rank, peer-mapped; [2][kTpMaxRanks] uint32
    int n_ranks, n_src, my_rank;
    __nv_bfloat16* x_shard;              // this rank's rows of the residual stream [nrows, d] (local)
    const __nv_bfloat16* w;              // norm weight [d] (local)
    int row0, nrows, d;
    float eps;
    uint32_t epoch;
    unsigned int* done_counter;          // local, zero between launches
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// data written by a peer GPU into this GPU's memory must not be served from this SM's (incoherent) L1: volatile 16-byte load
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void tp_wait_flags(const uint32_t* flags_local, int phase, int n_ranks, uint32_t epoch) {
    if ((int)threadIdx.x < n_ranks) {
        const uint32_t* f = flags_local + phase * kTpMaxRanks + threadIdx.x;
        uint32_t spins = 0;
        while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) {
            if (++spins > (1u << 27)) {
                printf("mmdp: tensor-parallel flag wait timeout (phase %d, source rank %d, epoch %u)\n", phase, (int)threadIdx.x, epoch);
                __trap();
            }
        }
    }
    __syncthreads();
}

// destination of the FP8 form: every rank's e4m3 activation buffer and its scales (peer-mapped)
struct TpFp8Out {
    uint8_t* q[kTpMaxRanks];  // [rows, d] e4m3
    float* s[kTpMaxRanks];    // [d / 128][ld_s] fp32, row index contiguous (the layout of quantize_fp8)
    int ld_s;
};

// d <= 2048 * NV columns (d % 8 == 0; d % 128 == 0 for F8): every thread owns up to NV groups of 8 consecutive columns
template <int NV, bool F8>
__device__ __forceinline__ void tp_reduce_norm_body(const TpReduceArgs& a, const TpFp8Out& f) {
    const int tid = threadIdx.x;
    // the phase-0 rendezvous (every rank's partial sums are complete) has been passed by tp_rendezvous_kernel, the previous
    // launch in this stream: this grid never spins
    pdl_launch_dependents();
    pdl_wait();
    const int lrow = blockIdx.x;
    const size_t grow = (size_t)(a.row0 + lrow) * a.d;
    __nv_bfloat16* xrow = a.x_shard + (size_t)lrow * a.d;
    float xv[NV][8];
    float ss = 0.f;
#pragma unroll
    for (int t = 0; t < NV; ++t) {
        const int c = (tid + t * kTpThreads) * 8;
        if (c >= a.d) {
#pragma unroll
            for (int j = 0; j < 8; ++j) xv[t][j] = 0.f;
            continue;
        }
        const uint4 xo = *reinterpret_cast<const uint4*>(xrow + c);
        const uint32_t xu[4] = {xo.x, xo.y, xo.z, xo.w};
        float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (a.n_src > 0) {
            float4 p0[kTpMaxRanks], p1[kTpMaxRanks];
#pragma unroll
            for (int r = 0; r < kTpMaxRanks; ++r)
                if (r < a.n_src) {
                    p0[r] = ld_peer_f4(a.part[r] + (size_t)lrow * a.d + c);
                    p1[r] = ld_peer_f4(a.part[r] + (size_t)lrow * a.d + c + 4);
                }
#pragma unroll
            for (int r = 0; r < kTpMaxRanks; ++r)
                if (r < a.n_src) {  // fixed rank order: the same sum on every rank and in every run
                    s[0] = __fadd_rn(s[0], p0[r].x); s[1] = __fadd_rn(s[1], p0[r].y); s[2] = __fadd_rn(s[2], p0[r].z); s[3] = __fadd_rn(s[3], p0[r].w);
                    s[4] = __fadd_rn(s[4], p1[r].x); s[5] = __fadd_rn(s[5], p1[r].y); s[6] = __fadd_rn(s[6], p1[r].z); s[7] = __fadd_rn(s[7], p1[r].w);
                }
        }
        uint32_t xw[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float lo = bf16_lo(xu[j]), hi = bf16_hi(xu[j]);
            if (a.n_src > 0) {  // x = bf16( bf16(linear output) + x )
                lo = bf16_round(__fadd_rn(lo, bf16_round(s[2 * j])));
                hi = bf16_round(__fadd_rn(hi, bf16_round(s[2 * j + 1])));
            }
            xv[t][2 * j] = lo;
            xv[t][2 * j + 1] = hi;
            ss = fmaf(lo, lo, ss);
            ss = fmaf(hi, hi, ss);
            xw[j] = pack_bf16x2(lo, hi);
        }
        if (a.n_src > 0) *reinterpret_cast<uint4*>(xrow + c) = make_uint4(xw[0], xw[1], xw[2], xw[3]);
    }
    __shared__ float red[kTpThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < kTpThreads / 32; ++i) tot += red[i];
    const float rstd = __frcp_rn(__fsqrt_rn(__fadd_rn(tot / (float)a.d, a.eps)));
#pragma unroll
    for (int t = 0; t < NV; ++t) {
        const int c = (tid + t * kTpThreads) * 8;
        if (c >= a.d) continue;
        const uint4 wv = *reinterpret_cast<const uint4*>(a.w + c);
        const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float n0 = bf16_round(__fmul_rn(xv[t][2 * j], rstd));
            const float n1 = bf16_round(__fmul_rn(xv[t][2 * j + 1], rstd));
            o[j] = pack_bf16x2(__fmul_rn(bf16_lo(ww[j]), n0), __fmul_rn(bf16_hi(ww[j]), n1));
        }
        if constexpr (F8) {
            // quantize_fp8_g128_kernel's arithmetic on the bf16 row: half-warp h of the warp holds one 128-column group
            const uint2 v0 = make_uint2(o[0], o[1]), v1 = make_uint2(o[2], o[3]);
            float amax = absmax4(v1, absmax4(v0, 0.f));
            const unsigned half_mask = 0xffffu << (tid & 16);
#pragma unroll
            for (int sh = 8; sh > 0; sh >>= 1) amax = fmaxf(amax, __shfl_xor_sync(half_mask, amax, sh));
            const float sc = amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f;
            const uint2 qv = make_uint2(quant4(v0, sc), quant4(v1, sc));
            const size_t si = (size_t)(c >> 7) * f.ld_s + a.row0 + lrow;
#pragma unroll
            for (int r = 0; r < kTpMaxRanks; ++r)
                if (r < a.n_ranks) {  // the all-gather of the e4m3 row and its scales: P2P stores
                    *reinterpret_cast<uint2*>(f.q[r] + grow + c) = qv;
                    if ((tid & 15) == 0) f.s[r][si] = sc;
                }
        } else {
            const uint4 ov = make_uint4(o[0], o[1], o[2], o[3]);
#pragma unroll
            for (int r = 0; r < kTpMaxRanks; ++r)
                if (r < a.n_ranks) *reinterpret_cast<uint4*>(a.xn[r] + grow + c) = ov;  // the all-gather: P2P stores
        }
    }
    // phase 1: when the LAST CTA of this rank has stored its rows, tell every rank that this rank's rows have landed
    __threadfence_system();
    __syncthreads();
    __shared__ int s_last;
    if (tid == 0) {
        const unsigned int prev = atomicAdd(a.done_counter, 1u);
        s_last = prev == (unsigned int)a.nrows - 1;
        if (s_last) *a.done_counter = 0;
    }
    __syncthreads();
    if (s_last && tid < a.n_ranks) st_release_sys(a.flags[tid] + 1 * kTpMaxRanks + a.my_rank, a.epoch);
}

template <int NV>
__global__ void __launch_bounds__(kTpThreads) tp_reduce_norm_kernel(TpReduceArgs a) {
    tp_reduce_norm_body<NV, false>(a, TpFp8Out{});
}

template <int NV>
__global__ void __launch_bounds__(kTpThreads) tp_reduce_norm_fp8_kernel(TpReduceArgs a, TpFp8Out f) {
    tp_reduce_norm_body<NV, true>(a, f);
}

// Phase 0 of a collective, ONE small CTA: tell every rank that this rank has reached the collective - its partial sums are
// complete (this kernel follows the producing GEMM in stream order) and it no longer reads the activation buffer the peers are
// about to overwrite - then wait for everybody's. The rendezvous is a kernel of its own so that nothing that spins on a
// peer holds more than 32 threads of this GPU: with two row chunks in flight, a 600-CTA reduce grid spinning on chunk A's
// flags filled the register files and kept chunk B's GEMM - which the PEER's chunk-B wait depended on - from starting
// (cross-rank deadlock, found by the flag-wait timeout at TP=2).
struct TpFlagPtrs { uint32_t* f[kTpMaxRanks]; };
__global__ void tp_rendezvous_kernel(TpFlagPtrs flags, int my_rank, int n_ranks, uint32_t epoch) {
    pdl_wait();
    if ((int)threadIdx.x < n_ranks) st_release_sys(flags.f[threadIdx.x] + 0 * kTpMaxRanks + my_rank, epoch);
    tp_wait_flags(flags.f[my_rank], 0, n_ranks, epoch);
    // only now may the dependent grid be scheduled: launched early it would sit at its griddepcontrol.wait holding registers
    // and shared memory on every SM while this CTA spins on the peers (the same starvation as a spinning grid)
    pdl_launch_dependents();
}

__global__ void tp_wait_kernel(const uint32_t* flags_local, int phase, int n_ranks, uint32_t epoch) {
    pdl_wait();
    tp_wait_flags(flags_local, phase, n_ranks, epoch);
    pdl_launch_dependents();  // after the wait, see tp_rendezvous_kernel
}

// f8 == nullptr: the bf16 form (xn); otherwise the FP8 form into f8's buffers (xn unused)
static int tp_reduce_launch(const float* recv_local, int rows_per_rank, int n_src, uint16_t* const* xn, const TpFp8Out* f8,
                            uint32_t* const* flags, int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* w, int row0, int nrows,
                            int d, float eps, uint32_t epoch, unsigned int* done_counter, cudaStream_t stream) {
    if (n_ranks < 1 || n_ranks > kTpMaxRanks || my_rank < 0 || my_rank >= n_ranks) return set_error("tp_reduce_norm: bad rank layout");
    if (n_src != 0 && n_src != n_ranks) return set_error("tp_reduce_norm: n_src must be 0 (no partial sums) or n_ranks");
    if (n_src && (!recv_local || nrows > rows_per_rank)) return set_error("tp_reduce_norm: receive buffer / rows_per_rank mismatch");
    if (nrows <= 0) return set_error("tp_reduce_norm: every rank must own at least one row (M >= n_ranks)");
    if (d % 8 || d > 8192) return set_error("tp_reduce_norm: d must be a multiple of 8 and <= 8192");
    TpReduceArgs a{};
    for (int r = 0; r < n_ranks; ++r) {
        a.part[r] = n_src ? recv_local + (size_t)r * rows_per_rank * d : nullptr;
        a.xn[r] = f8 ? nullptr : reinterpret_cast<__nv_bfloat16*>(xn[r]);
        a.flags[r] = flags[r];
    }
    a.n_ranks = n_ranks; a.n_src = n_src; a.my_rank = my_rank;
    a.x_shard = reinterpret_cast<__nv_bfloat16*>(x_shard);
    a.w = reinterpret_cast<const __nv_bfloat16*>(w);
    a.row0 = row0; a.nrows = nrows; a.d = d; a.eps = eps; a.epoch = epoch; a.done_counter = done_counter;
    const bool pdl = pdl_mode() != 0;
    cudaError_t e;
    {
        TpFlagPtrs fp{};
        for (int r = 0; r < n_ranks; ++r) fp.f[r] = flags[r];
        LaunchScope ls0(LK_ROW, 0.0, stream);
        MMDP_CUDA(launch_ex(tp_rendezvous_kernel, dim3(1), dim3(32), 0, stream, pdl, false, fp, my_rank, n_ranks, epoch));
    }
    {
    // bytes this rank moves: reads n_src fp32 rows + x, writes x + n_ranks bf16 rows (FP8: n_ranks e4m3 rows + their scales)
    const double out_row = f8 ? d + d / 32.0 : 2.0 * d;
    LaunchScope ls(LK_ROW, (double)nrows * (d * (4.0 * n_src + 4.0) + out_row * n_ranks), stream);
    const int nv = (d + 2047) / 2048;
    if (f8) {
        const TpFp8Out& f = *f8;
        switch (nv) {
            case 1: e = launch_ex(tp_reduce_norm_fp8_kernel<1>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a, f); break;
            case 2: e = launch_ex(tp_reduce_norm_fp8_kernel<2>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a, f); break;
            case 3: e = launch_ex(tp_reduce_norm_fp8_kernel<3>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a, f); break;
            default: e = launch_ex(tp_reduce_norm_fp8_kernel<4>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a, f); break;
        }
    } else {
        switch (nv) {
            case 1: e = launch_ex(tp_reduce_norm_kernel<1>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a); break;
            case 2: e = launch_ex(tp_reduce_norm_kernel<2>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a); break;
            case 3: e = launch_ex(tp_reduce_norm_kernel<3>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a); break;
            default: e = launch_ex(tp_reduce_norm_kernel<4>, dim3(nrows), dim3(kTpThreads), 0, stream, pdl, false, a); break;
        }
    }
    }
    MMDP_CUDA(e);
    // the consumer of xn (the next column-parallel GEMM) needs every rank's rows: wait for phase 1 of all ranks
    LaunchScope ls2(LK_ROW, 0.0, stream);
    MMDP_CUDA(launch_ex(tp_wait_kernel, dim3(1), dim3(32), 0, stream, pdl, false, (const uint32_t*)flags[my_rank], 1, n_ranks, epoch));
    return 0;
}

int tp_reduce_norm(const float* recv_local, int rows_per_rank, int n_src, uint16_t* const* xn, uint32_t* const* flags, int n_ranks,
                   int my_rank, uint16_t* x_shard, const uint16_t* w, int row0, int nrows, int d, float eps, uint32_t epoch,
                   unsigned int* done_counter, cudaStream_t stream) {
    return tp_reduce_launch(recv_local, rows_per_rank, n_src, xn, nullptr, flags, n_ranks, my_rank, x_shard, w, row0, nrows, d, eps,
                            epoch, done_counter, stream);
}

int tp_reduce_norm_fp8(const float* recv_local, int rows_per_rank, int n_src, uint8_t* const* xq, float* const* xs, int ld_s,
                       uint32_t* const* flags, int n_ranks, int my_rank, uint16_t* x_shard, const uint16_t* w, int row0, int nrows,
                       int d, float eps, uint32_t epoch, unsigned int* done_counter, cudaStream_t stream) {
    if (!xq || !xs) return set_error("tp_reduce_norm_fp8: null buffer array");
    if (d % 128) return set_error("tp_reduce_norm_fp8: d must be a multiple of 128 (the activation scale group)");
    if (ld_s < row0 + nrows) return set_error("tp_reduce_norm_fp8: the scale stride %d is below the rows %d", ld_s, row0 + nrows);
    if (n_ranks < 1 || n_ranks > kTpMaxRanks) return set_error("tp_reduce_norm: bad rank layout");
    TpFp8Out f{};
    for (int r = 0; r < n_ranks; ++r) {
        if (!xq[r] || !xs[r]) return set_error("tp_reduce_norm_fp8: null buffer of rank %d", r);
        f.q[r] = xq[r];
        f.s[r] = xs[r];
    }
    f.ld_s = ld_s;
    return tp_reduce_launch(recv_local, rows_per_rank, n_src, nullptr, &f, flags, n_ranks, my_rank, x_shard, w, row0, nrows, d, eps,
                            epoch, done_counter, stream);
}

}  // namespace mmdp
