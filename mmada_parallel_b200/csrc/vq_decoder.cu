// Native MagViT-v2 / VQGAN decoder context (MAGVITv2.decode_code, MMaDA-Parallel-M/models/modeling_magvitv2.py:429-433;
// VQGANDecoder.forward :365-399; ResnetBlock / AttnBlock / Upsample / Normalize in models/common_modules.py).
// Weights are repacked once: conv OIHW -> [tap][Cout][Cin padded to 32] fp32 so every convolution is one launch of the
// TF32 shifted-tap GEMM (conv_tf32.cu). Activations are fp32 channels-last with a one-pixel zero border.
#include "../../include/mmdp.h"
#include "mmdp_internal.h"

#include <map>
#include <string>
#include <vector>

using namespace mmdp;

struct ConvW {
    float* w = nullptr;     // [T][Cout][Kpad]
    float* bias = nullptr;  // [Cout]
    int cout = 0, cin = 0, kpad = 0, taps = 0;
    bool have_w = false, have_b = false;
};
struct NormW {
    float* gamma = nullptr;
    float* beta = nullptr;
    int c = 0;
    bool have_g = false, have_b = false;
};

// Sub-module names of a resnet / attention block: the taming-transformers layout of MagViT and diffusers' layout of the
// aMUSEd VQ-VAE. Registration and the forward helpers look names up through this table, so one code path serves both.
struct VqNames {
    const char* shortcut;   // 1x1 convolution of a resnet whose channel count changes
    const char* attn_norm;  // GroupNorm of the mid-block attention
    const char* q;
    const char* k;
    const char* v;
    const char* proj;       // output projection
};
static const VqNames kTamingNames = {".nin_shortcut", ".norm", ".q", ".k", ".v", ".proj_out"};
static const VqNames kDiffusersNames = {".conv_shortcut", ".group_norm", ".to_q", ".to_k", ".to_v", ".to_out.0"};

struct mmdp_vqdec {
    mmdp_vqdec_config cfg;
    const VqNames* names = &kTamingNames;
    // aMUSEd VQModel contexts only (mmdp_vqmodel_create)
    bool is_vqmodel = false;
    mmdp_vqmodel_config vm{};
    float* codebook = nullptr;  // [num_vq_embeddings][latent_channels]
    bool have_codebook = false;
    int* err = nullptr;         // device: bit 0 = id outside the codebook
    std::map<std::string, ConvW> conv;
    std::map<std::string, NormW> norm;
    std::vector<void*> allocs;
    float* buf[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t buf_elems = 0;
    float *q = nullptr, *k = nullptr, *vt = nullptr, *s = nullptr, *o = nullptr;
    double* stats = nullptr;
    float* stage = nullptr;  // raw-weight staging for packing
    size_t stage_elems = 0;
};

static int round32(int c) { return (c + 31) / 32 * 32; }

static int vq_alloc(mmdp_vqdec* d, void** p, size_t bytes) {
    if (cudaMalloc(p, bytes) != cudaSuccess) return set_error("vqdec: cudaMalloc(%zu) failed", bytes);
    if (cudaMemset(*p, 0, bytes) != cudaSuccess) return set_error("vqdec: cudaMemset failed");
    d->allocs.push_back(*p);
    return 0;
}

__global__ void pack_conv_kernel(const float* __restrict__ src, float* __restrict__ dst, int cout, int cin, int k, int kpad,
                                 int round_tf32) {
    // src OIHW [cout][cin][k][k] -> dst [t = ky*k+kx][cout][kpad]. round_tf32: store the weight rounded to the nearest TF32
    // value (tf32 wgmma otherwise drops the low 13 mantissa bits, a bias of half a TF32 ulp toward zero on every product)
    const long long n = (long long)k * k * cout * kpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % kpad);
        const int co = (int)((i / kpad) % cout);
        const int t = (int)(i / ((long long)kpad * cout));
        float v = ci < cin ? src[((size_t)co * cin + ci) * k * k + t] : 0.f;
        if (round_tf32) {
            uint32_t u;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
            v = __uint_as_float(u);
        }
        dst[i] = v;
    }
}

static int add_conv(mmdp_vqdec* d, const std::string& name, int cout, int cin, int k) {
    ConvW c;
    c.cout = cout; c.cin = cin; c.kpad = round32(cin); c.taps = k * k;
    if (vq_alloc(d, (void**)&c.w, (size_t)c.taps * cout * c.kpad * 4)) return -1;
    if (vq_alloc(d, (void**)&c.bias, (size_t)cout * 4)) return -1;
    d->conv[name] = c;
    const size_t raw = (size_t)cout * cin * k * k;
    if (raw > d->stage_elems) d->stage_elems = raw;
    return 0;
}
static int add_norm(mmdp_vqdec* d, const std::string& name, int c) {
    NormW n;
    n.c = c;
    if (vq_alloc(d, (void**)&n.gamma, (size_t)c * 4)) return -1;
    if (vq_alloc(d, (void**)&n.beta, (size_t)c * 4)) return -1;
    d->norm[name] = n;
    return 0;
}
static int add_resblock(mmdp_vqdec* d, const std::string& name, int cin, int cout) {
    if (add_norm(d, name + ".norm1", cin) || add_conv(d, name + ".conv1", cout, cin, 3) || add_norm(d, name + ".norm2", cout) ||
        add_conv(d, name + ".conv2", cout, cout, 3))
        return -1;
    if (cin != cout && add_conv(d, name + d->names->shortcut, cout, cin, 1)) return -1;
    return 0;
}
static int add_attn(mmdp_vqdec* d, const std::string& name, int c) {
    const VqNames& nm = *d->names;
    if (add_norm(d, name + nm.attn_norm, c)) return -1;
    for (const char* n : {nm.q, nm.k, nm.v, nm.proj})
        if (add_conv(d, name + n, c, c, 1)) return -1;
    return 0;
}

extern "C" {

MMDP_API int mmdp_vqdec_create(const mmdp_vqdec_config* c, mmdp_vqdec** out) {
    if (!c || !out) return set_error("mmdp_vqdec_create: null argument");
    if (c->n_levels < 1 || c->n_levels > 8 || c->ch % 32 || c->z_channels < 1 || c->z_channels > 32 || c->out_ch < 1 ||
        c->max_batch < 1 || c->latent_h < 1 || c->latent_w < 1)
        return set_error("mmdp_vqdec_create: bad config (ch must be a multiple of 32, n_levels in [1,8])");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return set_error("mmdp_vqdec_create: no CUDA device (this library has no CPU fallback)");
    mmdp_vqdec* d = new mmdp_vqdec();
    d->cfg = *c;
    const int nres = c->n_levels;
    int block_in = c->ch * c->ch_mult[nres - 1];
    int rc = 0;
    rc |= add_conv(d, "decoder.post_quant_conv", c->z_channels, c->z_channels, 1);
    rc |= add_conv(d, "decoder.conv_in", block_in, c->z_channels, 3);
    rc |= add_resblock(d, "decoder.mid.block_1", block_in, block_in);
    rc |= add_attn(d, "decoder.mid.attn_1", block_in);
    rc |= add_resblock(d, "decoder.mid.block_2", block_in, block_in);
    int H = c->latent_h, W = c->latent_w;
    size_t max_elems = (size_t)(H + 2) * (W + 2) * block_in;
    for (int lvl = nres - 1; lvl >= 0; --lvl) {
        const int block_out = c->ch * c->ch_mult[lvl];
        for (int b = 0; b < c->num_res_blocks[lvl]; ++b) {
            rc |= add_resblock(d, "decoder.up." + std::to_string(lvl) + ".block." + std::to_string(b), block_in, block_out);
            const size_t e = (size_t)(H + 2) * (W + 2) * (block_in > block_out ? block_in : block_out);
            if (e > max_elems) max_elems = e;
            block_in = block_out;
        }
        if (lvl != 0) {
            rc |= add_conv(d, "decoder.up." + std::to_string(lvl) + ".upsample.conv", block_in, block_in, 3);
            H *= 2; W *= 2;
            const size_t e = (size_t)(H + 2) * (W + 2) * block_in;
            if (e > max_elems) max_elems = e;
        }
    }
    rc |= add_norm(d, "decoder.norm_out", block_in);
    rc |= add_conv(d, "decoder.conv_out", c->out_ch, block_in, 3);
    d->buf_elems = max_elems * c->max_batch;
    for (int i = 0; i < 4; ++i) rc |= vq_alloc(d, (void**)&d->buf[i], d->buf_elems * 4);
    const size_t hw = (size_t)c->latent_h * c->latent_w;
    const int cm = c->ch * c->ch_mult[nres - 1];
    rc |= vq_alloc(d, (void**)&d->q, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->k, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->o, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->vt, (size_t)cm * round32((int)hw) * 4);
    rc |= vq_alloc(d, (void**)&d->s, hw * round32((int)hw) * 4);
    rc |= vq_alloc(d, (void**)&d->stats, (size_t)c->max_batch * 32 * 2 * sizeof(double));
    rc |= vq_alloc(d, (void**)&d->stage, d->stage_elems * 4);
    if (rc) {
        mmdp_vqdec_destroy(d);
        return -1;
    }
    *out = d;
    return 0;
}

MMDP_API void mmdp_vqdec_destroy(mmdp_vqdec* d) {
    if (!d) return;
    for (void* p : d->allocs) cudaFree(p);
    delete d;
}

MMDP_API int mmdp_vqdec_set_weight(mmdp_vqdec* d, const char* name, const float* src, int64_t numel, void* stream) {
    if (!d || !name || !src) return set_error("mmdp_vqdec_set_weight: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    std::string n(name);
    const bool is_w = n.size() > 7 && n.compare(n.size() - 7, 7, ".weight") == 0;
    const bool is_b = n.size() > 5 && n.compare(n.size() - 5, 5, ".bias") == 0;
    if (!is_w && !is_b) return set_error("mmdp_vqdec_set_weight: '%s' is neither .weight nor .bias", name);
    const std::string base = n.substr(0, n.size() - (is_w ? 7 : 5));
    if (d->codebook && n == "quantize.embedding.weight") {
        const int64_t want = (int64_t)d->vm.num_vq_embeddings * d->vm.latent_channels;
        if (numel != want) return set_error("mmdp_vqdec_set_weight(%s): expected %lld elements, got %lld", name, (long long)want, (long long)numel);
        MMDP_CUDA(cudaMemcpyAsync(d->codebook, src, (size_t)want * 4, cudaMemcpyDefault, s));
        d->have_codebook = true;
        return 0;
    }
    auto ci = d->conv.find(base);
    if (ci != d->conv.end()) {
        ConvW& c = ci->second;
        if (is_b) {
            if (numel != c.cout) return set_error("mmdp_vqdec_set_weight(%s): expected %d elements, got %lld", name, c.cout, (long long)numel);
            MMDP_CUDA(cudaMemcpyAsync(c.bias, src, (size_t)c.cout * 4, cudaMemcpyDefault, s));
            c.have_b = true;
            return 0;
        }
        const int k = c.taps == 9 ? 3 : 1;
        const int64_t want = (int64_t)c.cout * c.cin * c.taps;
        if (numel != want) return set_error("mmdp_vqdec_set_weight(%s): expected %lld elements, got %lld", name, (long long)want, (long long)numel);
        MMDP_CUDA(cudaMemcpyAsync(d->stage, src, (size_t)want * 4, cudaMemcpyDefault, s));
        pack_conv_kernel<<<256, 256, 0, s>>>(d->stage, c.w, c.cout, c.cin, k, c.kpad, d->is_vqmodel ? 1 : 0);
        MMDP_CUDA(cudaGetLastError());
        MMDP_CUDA(cudaStreamSynchronize(s));  // the staging buffer is reused by the next call
        c.have_w = true;
        return 0;
    }
    auto ni = d->norm.find(base);
    if (ni != d->norm.end()) {
        NormW& nw = ni->second;
        if (numel != nw.c) return set_error("mmdp_vqdec_set_weight(%s): expected %d elements, got %lld", name, nw.c, (long long)numel);
        MMDP_CUDA(cudaMemcpyAsync(is_w ? nw.gamma : nw.beta, src, (size_t)nw.c * 4, cudaMemcpyDefault, s));
        (is_w ? nw.have_g : nw.have_b) = true;
        return 0;
    }
    return set_error("mmdp_vqdec_set_weight: unknown parameter '%s'", name);
}

MMDP_API int mmdp_vqdec_missing(mmdp_vqdec* d, char* out, int out_len) {
    if (!d) return -1;
    std::string m;
    int count = 0;
    for (auto& kv : d->conv) {
        if (!kv.second.have_w) { m += kv.first + ".weight "; ++count; }
        if (!kv.second.have_b) { m += kv.first + ".bias "; ++count; }
    }
    for (auto& kv : d->norm) {
        if (!kv.second.have_g) { m += kv.first + ".weight "; ++count; }
        if (!kv.second.have_b) { m += kv.first + ".bias "; ++count; }
    }
    if (d->codebook && !d->have_codebook) { m += "quantize.embedding.weight "; ++count; }
    if (out && out_len > 0) snprintf(out, (size_t)out_len, "%s", m.c_str());
    return count;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
namespace {

struct Fwd {
    mmdp_vqdec* d;
    cudaStream_t s;
    int B;

    int conv(const std::string& name, const float* x, int H, int W, float* y, const float* resid) {
        const ConvW& c = d->conv.at(name);
        const int Hp = H + 2, Wp = W + 2;
        const int M = B * Hp * Wp;
        int shifts[9];
        if (c.taps == 9)
            for (int ky = 0; ky < 3; ++ky)
                for (int kx = 0; kx < 3; ++kx) shifts[ky * 3 + kx] = (ky - 1) * Wp + (kx - 1);
        else
            shifts[0] = 0;
        // activations carry round32(cin) channels per pixel (zero beyond cin); outputs are written with ld = round32(cout)
        return conv_tf32(x, c.kpad, M, c.w, M, c.cout, c.kpad, c.taps, shifts, y, round32(c.cout), resid, round32(c.cout), c.bias,
                         0, 1.0f, Wp, Hp, 0, 0, s);
    }
    int gn(const std::string& name, const float* x, float* y, int H, int W, int swish, int compact) {
        const NormW& n = d->norm.at(name);
        return gn_swish(x, y, B, n.c, H, W, d->stats, n.gamma, n.beta, 1e-6f, swish, compact, s);
    }
    // ResnetBlock.forward (common_modules.py:335-357), temb None: x in buf[ix] -> result in buf[iy]
    int resblock(const std::string& name, int H, int W, int& ix) {
        float* X = d->buf[ix];
        float* T = d->buf[(ix + 1) & 3];
        float* Hb = d->buf[(ix + 2) & 3];
        float* Y = d->buf[(ix + 3) & 3];
        if (gn(name + ".norm1", X, T, H, W, 1, 0)) return -1;
        if (conv(name + ".conv1", T, H, W, Hb, nullptr)) return -1;
        if (gn(name + ".norm2", Hb, T, H, W, 1, 0)) return -1;
        const float* res = X;
        const std::string sc = name + d->names->shortcut;
        if (d->conv.count(sc)) {
            if (conv(sc, X, H, W, Hb, nullptr)) return -1;  // Hb is free again after norm2
            res = Hb;
        }
        if (conv(name + ".conv2", T, H, W, Y, res)) return -1;
        ix = (ix + 3) & 3;
        return 0;
    }
    // AttnBlock.forward (common_modules.py:186-211); diffusers' single-head Attention of UNetMidBlock2D is the same math
    int attn(const std::string& name, int H, int W, int& ix) {
        const VqNames& nm = *d->names;
        float* X = d->buf[ix];
        float* T = d->buf[(ix + 1) & 3];
        float* Y = d->buf[(ix + 3) & 3];
        const int C = d->norm.at(name + nm.attn_norm).c, hw = H * W, hwp = round32(hw);
        if (gn(name + nm.attn_norm, X, T, H, W, 0, 1)) return -1;  // compact [B, hw, C]
        const ConvW& wq = d->conv.at(name + nm.q);
        const ConvW& wk = d->conv.at(name + nm.k);
        const ConvW& wv = d->conv.at(name + nm.v);
        const ConvW& wp = d->conv.at(name + nm.proj);
        if (conv_tf32(T, C, (long long)B * hw, wq.w, B * hw, C, C, 1, nullptr, d->q, C, nullptr, 0, wq.bias, 0, 1.f, 0, 0, 0, 0, s)) return -1;
        if (conv_tf32(T, C, (long long)B * hw, wk.w, B * hw, C, C, 1, nullptr, d->k, C, nullptr, 0, wk.bias, 0, 1.f, 0, 0, 0, 0, s)) return -1;
        const float scale = 1.0f / sqrtf((float)C);
        if (hwp != hw) {
            // P . V runs over hwp keys: the padding columns of S and V^T must be zero, also after a larger grid used them
            MMDP_CUDA(cudaMemsetAsync(d->s, 0, (size_t)hw * hwp * 4, s));
            MMDP_CUDA(cudaMemsetAsync(d->vt, 0, (size_t)C * hwp * 4, s));
        }
        for (int b = 0; b < B; ++b) {
            const float* hn = T + (size_t)b * hw * C;
            // V^T [C, hw] = Wv [C, C] . hn^T, bias along rows
            if (conv_tf32(wv.w, C, C, hn, C, hw, C, 1, nullptr, d->vt, hwp, nullptr, 0, wv.bias, 1, 1.f, 0, 0, 0, 0, s)) return -1;
            // S [hw, hw] = q k^T * C^-0.5
            if (conv_tf32(d->q + (size_t)b * hw * C, C, hw, d->k + (size_t)b * hw * C, hw, hw, C, 1, nullptr, d->s, hwp, nullptr, 0,
                          nullptr, 0, scale, 0, 0, 0, 0, s))
                return -1;
            if (softmax_rows_ld(d->s, hw, hw, hwp, s)) return -1;
            // O [hw, C] = P [hw, hw] . V   (W operand = V^T [C, hw]); K = hwp (padding columns of P and V^T are zero)
            if (conv_tf32(d->s, hwp, hw, d->vt, hw, C, hwp, 1, nullptr, d->o + (size_t)b * hw * C, C, nullptr, 0, nullptr, 0, 1.f, 0,
                          0, 0, 0, s))
                return -1;
        }
        // out = x + proj_out(O): compact rows scattered into the padded layout with the padded residual
        if (conv_tf32(d->o, C, (long long)B * hw, wp.w, B * hw, C, C, 1, nullptr, Y, C, X, C, wp.bias, 0, 1.f, 0, 0, W, H, s)) return -1;
        // the scatter writes interior pixels only: re-establish the zero border of Y
        if (zero_border(Y, B, C, H, W, s)) return -1;
        ix = (ix + 3) & 3;
        return 0;
    }
};

}  // namespace

extern "C" MMDP_API int mmdp_vqdec_decode(mmdp_vqdec* d, const int64_t* ids, int B, int h, int w, float* out_nchw, void* stream) {
    if (!d || !ids || !out_nchw) return set_error("mmdp_vqdec_decode: null argument");
    const mmdp_vqdec_config& c = d->cfg;
    if (d->is_vqmodel) return set_error("mmdp_vqdec_decode: a VQModel context decodes with mmdp_vqmodel_decode");
    if (B < 1 || B > c.max_batch || h != c.latent_h || w != c.latent_w)
        return set_error("mmdp_vqdec_decode: B=%d h=%d w=%d outside the context (max_batch=%d, latent %dx%d)", B, h, w, c.max_batch, c.latent_h, c.latent_w);
    char miss[256];
    if (mmdp_vqdec_missing(d, miss, sizeof(miss)) != 0) return set_error("mmdp_vqdec_decode: parameters not loaded: %s", miss);
    cudaStream_t s = (cudaStream_t)stream;
    Fwd f{d, s, B};
    int ix = 0, H = h, W = w;
    const int zc = round32(c.z_channels);
    // LFQuantizer.get_codebook_entry straight into the padded channels-last input
    MMDP_CUDA(cudaMemsetAsync(d->buf[0], 0, (size_t)B * (H + 2) * (W + 2) * zc * 4, s));
    if (lfq_to_padded(ids, d->buf[0], B, H, W, c.z_channels, zc, s)) return -1;
    MMDP_CUDA(cudaMemsetAsync(d->buf[1], 0, (size_t)B * (H + 2) * (W + 2) * zc * 4, s));  // channels z..31 of post_quant out stay 0
    if (f.conv("decoder.post_quant_conv", d->buf[0], H, W, d->buf[1], nullptr)) return -1;
    if (f.conv("decoder.conv_in", d->buf[1], H, W, d->buf[2], nullptr)) return -1;
    ix = 2;
    if (f.resblock("decoder.mid.block_1", H, W, ix)) return -1;
    if (f.attn("decoder.mid.attn_1", H, W, ix)) return -1;
    if (f.resblock("decoder.mid.block_2", H, W, ix)) return -1;
    for (int lvl = c.n_levels - 1; lvl >= 0; --lvl) {
        for (int b = 0; b < c.num_res_blocks[lvl]; ++b)
            if (f.resblock("decoder.up." + std::to_string(lvl) + ".block." + std::to_string(b), H, W, ix)) return -1;
        if (lvl != 0) {
            const int C = c.ch * c.ch_mult[lvl];
            float* X = d->buf[ix];
            float* T = d->buf[(ix + 1) & 3];
            float* Y = d->buf[(ix + 3) & 3];
            if (upsample2x(X, T, B, C, H, W, s)) return -1;
            H *= 2; W *= 2;
            if (f.conv("decoder.up." + std::to_string(lvl) + ".upsample.conv", T, H, W, Y, nullptr)) return -1;
            ix = (ix + 3) & 3;
        }
    }
    float* X = d->buf[ix];
    float* T = d->buf[(ix + 1) & 3];
    float* Y = d->buf[(ix + 3) & 3];
    if (f.gn("decoder.norm_out", X, T, H, W, 1, 0)) return -1;
    if (f.conv("decoder.conv_out", T, H, W, Y, nullptr)) return -1;
    return padded_to_nchw(Y, out_nchw, B, c.out_ch, round32(c.out_ch), H, W, s);
}

// ------------------------------------------------------------------------------------------------
// Encoder: MAGVITv2.get_code (modeling_magvitv2.py:423-427) = VQGANEncoder.forward (:143-169) + LFQ sign bits.
// Same net object type as the decoder (weights registry + rotating activation buffers); parameters are registered
// under the reference's 'encoder.*' names. Downsample (3x3, stride 2, pad (0,1,0,1)) = the stride-1 zero-border conv
// followed by picking input pixels (2y+1, 2x+1).
// ------------------------------------------------------------------------------------------------
extern "C" {

MMDP_API int mmdp_vqenc_create(const mmdp_vqdec_config* c, mmdp_vqdec** out) {
    if (!c || !out) return set_error("mmdp_vqenc_create: null argument");
    if (c->n_levels < 1 || c->n_levels > 8 || c->ch % 32 || c->z_channels < 1 || c->z_channels > 32 || c->out_ch < 1 ||
        c->out_ch > 32 || c->max_batch < 1 || c->latent_h < 1 || c->latent_w < 1)
        return set_error("mmdp_vqenc_create: bad config (out_ch = image channels; latent_h/w = code grid)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return set_error("mmdp_vqenc_create: no CUDA device (this library has no CPU fallback)");
    mmdp_vqdec* d = new mmdp_vqdec();
    d->cfg = *c;
    const int nres = c->n_levels;
    int rc = 0;
    int H = c->latent_h << (nres - 1), W = c->latent_w << (nres - 1);  // pixel resolution
    rc |= add_conv(d, "encoder.conv_in", c->ch, c->out_ch, 3);
    size_t max_elems = (size_t)(H + 2) * (W + 2) * c->ch;
    int block_in = c->ch;
    for (int lvl = 0; lvl < nres; ++lvl) {
        const int block_out = c->ch * c->ch_mult[lvl];
        for (int b = 0; b < c->num_res_blocks[lvl]; ++b) {
            rc |= add_resblock(d, "encoder.down." + std::to_string(lvl) + ".block." + std::to_string(b), block_in, block_out);
            const size_t e = (size_t)(H + 2) * (W + 2) * (block_in > block_out ? block_in : block_out);
            if (e > max_elems) max_elems = e;
            block_in = block_out;
        }
        if (lvl != nres - 1) {
            rc |= add_conv(d, "encoder.down." + std::to_string(lvl) + ".downsample.conv", block_in, block_in, 3);
            H /= 2; W /= 2;
        }
    }
    rc |= add_resblock(d, "encoder.mid.block_1", block_in, block_in);
    rc |= add_attn(d, "encoder.mid.attn_1", block_in);
    rc |= add_resblock(d, "encoder.mid.block_2", block_in, block_in);
    rc |= add_norm(d, "encoder.norm_out", block_in);
    rc |= add_conv(d, "encoder.conv_out", c->z_channels, block_in, 3);
    rc |= add_conv(d, "encoder.quant_conv", c->z_channels, c->z_channels, 1);
    d->buf_elems = max_elems * c->max_batch;
    for (int i = 0; i < 4; ++i) rc |= vq_alloc(d, (void**)&d->buf[i], d->buf_elems * 4);
    const size_t hw = (size_t)c->latent_h * c->latent_w;
    const int cm = block_in;
    rc |= vq_alloc(d, (void**)&d->q, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->k, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->o, (size_t)c->max_batch * hw * cm * 4);
    rc |= vq_alloc(d, (void**)&d->vt, (size_t)cm * round32((int)hw) * 4);
    rc |= vq_alloc(d, (void**)&d->s, hw * round32((int)hw) * 4);
    rc |= vq_alloc(d, (void**)&d->stats, (size_t)c->max_batch * 32 * 2 * sizeof(double));
    rc |= vq_alloc(d, (void**)&d->stage, d->stage_elems * 4);
    if (rc) {
        mmdp_vqdec_destroy(d);
        return -1;
    }
    *out = d;
    return 0;
}

MMDP_API int mmdp_vqenc_encode(mmdp_vqdec* d, const float* pixels_nchw, int B, int H, int W, int64_t* ids_out, void* stream) {
    if (!d || !pixels_nchw || !ids_out) return set_error("mmdp_vqenc_encode: null argument");
    if (d->is_vqmodel) return set_error("mmdp_vqenc_encode: a VQModel context encodes with mmdp_vqmodel_encode");
    const mmdp_vqdec_config& c = d->cfg;
    const int nres = c.n_levels;
    if (B < 1 || B > c.max_batch || H != (c.latent_h << (nres - 1)) || W != (c.latent_w << (nres - 1)))
        return set_error("mmdp_vqenc_encode: B=%d H=%d W=%d outside the context (max_batch=%d, %dx%d pixels)", B, H, W, c.max_batch,
                         c.latent_h << (nres - 1), c.latent_w << (nres - 1));
    if (!d->conv.count("encoder.conv_in")) return set_error("mmdp_vqenc_encode: not an encoder context");
    char miss[256];
    if (mmdp_vqdec_missing(d, miss, sizeof(miss)) != 0) return set_error("mmdp_vqenc_encode: parameters not loaded: %s", miss);
    cudaStream_t s = (cudaStream_t)stream;
    Fwd f{d, s, B};
    const int cin = round32(c.out_ch);
    if (nchw_to_padded(pixels_nchw, d->buf[0], B, c.out_ch, cin, H, W, s)) return -1;
    if (f.conv("encoder.conv_in", d->buf[0], H, W, d->buf[1], nullptr)) return -1;
    int ix = 1;
    for (int lvl = 0; lvl < nres; ++lvl) {
        for (int b = 0; b < c.num_res_blocks[lvl]; ++b)
            if (f.resblock("encoder.down." + std::to_string(lvl) + ".block." + std::to_string(b), H, W, ix)) return -1;
        if (lvl != nres - 1) {
            const int C = c.ch * c.ch_mult[lvl];
            float* X = d->buf[ix];
            float* T = d->buf[(ix + 1) & 3];
            float* Y = d->buf[(ix + 3) & 3];
            if (f.conv("encoder.down." + std::to_string(lvl) + ".downsample.conv", X, H, W, T, nullptr)) return -1;
            if (downsample_pick(T, Y, B, C, H, W, s)) return -1;
            H /= 2; W /= 2;
            ix = (ix + 3) & 3;
        }
    }
    if (f.resblock("encoder.mid.block_1", H, W, ix)) return -1;
    if (f.attn("encoder.mid.attn_1", H, W, ix)) return -1;
    if (f.resblock("encoder.mid.block_2", H, W, ix)) return -1;
    float* X = d->buf[ix];
    float* T = d->buf[(ix + 1) & 3];
    float* Y = d->buf[(ix + 3) & 3];
    if (f.gn("encoder.norm_out", X, T, H, W, 1, 0)) return -1;
    const int zc = round32(c.z_channels);
    MMDP_CUDA(cudaMemsetAsync(Y, 0, (size_t)B * (H + 2) * (W + 2) * zc * 4, s));  // channels z..31 stay zero (quant_conv input)
    if (f.conv("encoder.conv_out", T, H, W, Y, nullptr)) return -1;
    if (f.conv("encoder.quant_conv", Y, H, W, X, nullptr)) return -1;
    return lfq_indices(X, ids_out, B, H, W, c.z_channels, zc, s);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// aMUSEd VQ-VAE: diffusers.VQModel (autoencoders/vq_model.py) with Encoder / Decoder of autoencoders/vae.py, blocks of
// unets/unet_2d_blocks.py (DownEncoderBlock2D, UpDecoderBlock2D, UNetMidBlock2D), resnet.py (ResnetBlock2D),
// downsampling.py / upsampling.py. The same weight registry, Fwd helpers and rotating buffers as the MagViT contexts, under
// diffusers' names (kDiffusersNames) and for any latent grid of at most max_latent_cells cells.
// ------------------------------------------------------------------------------------------------
namespace {

// Largest padded area (H+2)(W+2) of a grid h x w with h*w <= cells at s pixels per cell:
// hw s^2 + 2s(h+w) + 4 with h + w <= hw + 1, reached by the 1 x cells grid.
size_t worst_padded(int cells, int s) { return (size_t)((long long)cells * s + 2) * (size_t)(s + 2); }

int mid_block(Fwd& f, const std::string& name, int H, int W, int& ix, bool attn) {
    if (f.resblock(name + ".resnets.0", H, W, ix)) return -1;
    if (attn && f.attn(name + ".attentions.0", H, W, ix)) return -1;
    return f.resblock(name + ".resnets.1", H, W, ix);
}

std::string blk(const char* prefix, int i, const char* mid, int j) {
    return std::string(prefix) + std::to_string(i) + mid + std::to_string(j);
}

}  // namespace

extern "C" {

MMDP_API int mmdp_vqmodel_create(const mmdp_vqmodel_config* c, mmdp_vqdec** out) {
    if (!c || !out) return set_error("mmdp_vqmodel_create: null argument");
    const int L = c->n_levels;
    if (L < 1 || L > 8) return set_error("mmdp_vqmodel_create: n_levels=%d outside [1, 8]", L);
    for (int i = 0; i < L; ++i)
        if (c->block_out_channels[i] < 32 || c->block_out_channels[i] % 32)
            return set_error("mmdp_vqmodel_create: block_out_channels[%d]=%d is not a positive multiple of 32 (GroupNorm with 32 groups "
                             "on float4 rows)", i, c->block_out_channels[i]);
    if (c->latent_channels < 1 || c->latent_channels > 256)
        return set_error("mmdp_vqmodel_create: latent_channels=%d outside [1, 256]", c->latent_channels);
    if (c->in_channels < 1 || c->in_channels > 32 || c->out_channels < 1 || c->out_channels > 32)
        return set_error("mmdp_vqmodel_create: in_channels=%d / out_channels=%d outside [1, 32]", c->in_channels, c->out_channels);
    if (c->layers_per_block < 1 || c->layers_per_block > 16)
        return set_error("mmdp_vqmodel_create: layers_per_block=%d outside [1, 16]", c->layers_per_block);
    if (c->num_vq_embeddings < 1) return set_error("mmdp_vqmodel_create: num_vq_embeddings=%d", c->num_vq_embeddings);
    if (c->max_batch < 1 || c->max_latent_cells < 1)
        return set_error("mmdp_vqmodel_create: max_batch=%d, max_latent_cells=%d must be >= 1", c->max_batch, c->max_latent_cells);
    const int smax = 1 << (L - 1);
    if ((double)c->max_batch * (double)worst_padded(c->max_latent_cells, smax) > 2.0e9)
        return set_error("mmdp_vqmodel_create: max_batch x max_latent_cells too large (padded pixel rows must fit in int32)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return set_error("mmdp_vqmodel_create: no CUDA device (this library has no CPU fallback)");
    mmdp_vqdec* d = new mmdp_vqdec();
    d->names = &kDiffusersNames;
    d->is_vqmodel = true;
    d->vm = *c;
    d->cfg.max_batch = c->max_batch;
    const int* boc = c->block_out_channels;
    const int top = boc[L - 1], lat = c->latent_channels, N = c->max_latent_cells, lpb = c->layers_per_block;
    const bool attn = c->mid_block_add_attention != 0;
    size_t max_elems = 0;
    auto need = [&](int s, int ch) {
        const size_t e = worst_padded(N, s) * (size_t)ch;
        if (e > max_elems) max_elems = e;
    };
    int rc = 0;
    // Encoder: conv_in -> down_blocks.i (layers_per_block resnets, downsamplers.0.conv except on the last) -> mid_block ->
    // conv_norm_out + SiLU -> conv_out (latent_channels) ; quant_conv
    rc |= add_conv(d, "encoder.conv_in", boc[0], c->in_channels, 3);
    need(smax, round32(c->in_channels));
    int cin = boc[0];
    for (int i = 0; i < L; ++i) {
        const int cout = boc[i], s = smax >> i;
        need(s, cin > cout ? cin : cout);
        for (int j = 0; j < lpb; ++j) {
            rc |= add_resblock(d, blk("encoder.down_blocks.", i, ".resnets.", j), j == 0 ? cin : cout, cout);
        }
        cin = cout;
        if (i != L - 1) rc |= add_conv(d, "encoder.down_blocks." + std::to_string(i) + ".downsamplers.0.conv", cout, cout, 3);
    }
    rc |= add_resblock(d, "encoder.mid_block.resnets.0", top, top);
    if (attn) rc |= add_attn(d, "encoder.mid_block.attentions.0", top);
    rc |= add_resblock(d, "encoder.mid_block.resnets.1", top, top);
    rc |= add_norm(d, "encoder.conv_norm_out", top);
    rc |= add_conv(d, "encoder.conv_out", lat, top, 3);
    rc |= add_conv(d, "quant_conv", lat, lat, 1);
    need(1, round32(lat) > top ? round32(lat) : top);
    // post_quant_conv ; Decoder: conv_in -> mid_block -> up_blocks.i in reversed channel order (layers_per_block + 1 resnets,
    // upsamplers.0.conv except on the last) -> conv_norm_out + SiLU -> conv_out
    rc |= add_conv(d, "post_quant_conv", lat, lat, 1);
    rc |= add_conv(d, "decoder.conv_in", top, lat, 3);
    rc |= add_resblock(d, "decoder.mid_block.resnets.0", top, top);
    if (attn) rc |= add_attn(d, "decoder.mid_block.attentions.0", top);
    rc |= add_resblock(d, "decoder.mid_block.resnets.1", top, top);
    cin = top;
    for (int i = 0; i < L; ++i) {
        const int cout = boc[L - 1 - i], s = 1 << i;
        need(s, cin > cout ? cin : cout);
        for (int j = 0; j <= lpb; ++j) rc |= add_resblock(d, blk("decoder.up_blocks.", i, ".resnets.", j), j == 0 ? cin : cout, cout);
        cin = cout;
        if (i != L - 1) {
            rc |= add_conv(d, "decoder.up_blocks." + std::to_string(i) + ".upsamplers.0.conv", cout, cout, 3);
            need(2 * s, cout);
        }
    }
    rc |= add_norm(d, "decoder.conv_norm_out", boc[0]);
    rc |= add_conv(d, "decoder.conv_out", c->out_channels, boc[0], 3);
    need(smax, round32(c->out_channels));
    d->buf_elems = max_elems * c->max_batch;
    for (int i = 0; i < 4; ++i) rc |= vq_alloc(d, (void**)&d->buf[i], d->buf_elems * 4);
    if (attn) {
        rc |= vq_alloc(d, (void**)&d->q, (size_t)c->max_batch * N * top * 4);
        rc |= vq_alloc(d, (void**)&d->k, (size_t)c->max_batch * N * top * 4);
        rc |= vq_alloc(d, (void**)&d->o, (size_t)c->max_batch * N * top * 4);
        rc |= vq_alloc(d, (void**)&d->vt, (size_t)top * round32(N) * 4);
        rc |= vq_alloc(d, (void**)&d->s, (size_t)N * round32(N) * 4);
    }
    rc |= vq_alloc(d, (void**)&d->stats, (size_t)c->max_batch * 32 * 2 * sizeof(double));
    rc |= vq_alloc(d, (void**)&d->codebook, (size_t)c->num_vq_embeddings * lat * 4);
    rc |= vq_alloc(d, (void**)&d->err, sizeof(int));
    const size_t cb_elems = (size_t)c->num_vq_embeddings * lat;
    if (cb_elems > d->stage_elems) d->stage_elems = cb_elems;
    rc |= vq_alloc(d, (void**)&d->stage, d->stage_elems * 4);
    if (rc) {
        mmdp_vqdec_destroy(d);
        return -1;
    }
    *out = d;
    return 0;
}

static int vqmodel_check(mmdp_vqdec* d, const char* fn, int B, int h, int w) {
    if (!d->is_vqmodel) return set_error("%s: not a VQModel context (create it with mmdp_vqmodel_create)", fn);
    const mmdp_vqmodel_config& c = d->vm;
    if (B < 1 || B > c.max_batch || h < 1 || w < 1 || (long long)h * w > c.max_latent_cells)
        return set_error("%s: B=%d, latent grid %dx%d outside the context (max_batch=%d, max_latent_cells=%d)", fn, B, h, w, c.max_batch,
                         c.max_latent_cells);
    char miss[256];
    if (mmdp_vqdec_missing(d, miss, sizeof(miss)) != 0) return set_error("%s: parameters not loaded: %s", fn, miss);
    return 0;
}

MMDP_API int mmdp_vqmodel_decode(mmdp_vqdec* d, const int64_t* ids, const float* latents_nchw, int B, int h, int w, float* out_nchw,
                                 void* stream) {
    if (!d || !out_nchw || (!ids == !latents_nchw))
        return set_error("mmdp_vqmodel_decode: null argument (exactly one of ids / latents must be given)");
    if (vqmodel_check(d, "mmdp_vqmodel_decode", B, h, w)) return -1;
    const mmdp_vqmodel_config& c = d->vm;
    cudaStream_t s = (cudaStream_t)stream;
    Fwd f{d, s, B};
    const int L = c.n_levels, lat = c.latent_channels, zc = round32(lat);
    const size_t zbytes = (size_t)B * (h + 2) * (w + 2) * zc * 4;
    if (ids) {
        // quantize.get_codebook_entry straight into the padded channels-last input
        MMDP_CUDA(cudaMemsetAsync(d->buf[0], 0, zbytes, s));
        if (codebook_to_padded(ids, d->codebook, d->buf[0], B, h, w, lat, zc, c.num_vq_embeddings, d->err, s)) return -1;
    } else if (nchw_to_padded(latents_nchw, d->buf[0], B, lat, zc, h, w, s)) {
        return -1;
    }
    MMDP_CUDA(cudaMemsetAsync(d->buf[1], 0, zbytes, s));  // channels lat..zc of post_quant_conv's output stay 0
    if (f.conv("post_quant_conv", d->buf[0], h, w, d->buf[1], nullptr)) return -1;
    if (f.conv("decoder.conv_in", d->buf[1], h, w, d->buf[2], nullptr)) return -1;
    int ix = 2, H = h, W = w;
    if (mid_block(f, "decoder.mid_block", H, W, ix, c.mid_block_add_attention != 0)) return -1;
    for (int i = 0; i < L; ++i) {
        for (int j = 0; j <= c.layers_per_block; ++j)
            if (f.resblock(blk("decoder.up_blocks.", i, ".resnets.", j), H, W, ix)) return -1;
        if (i != L - 1) {
            // Upsample2D: nearest 2x, then the 3x3 convolution
            const int C = c.block_out_channels[L - 1 - i];
            float* X = d->buf[ix];
            float* T = d->buf[(ix + 1) & 3];
            float* Y = d->buf[(ix + 3) & 3];
            if (upsample2x(X, T, B, C, H, W, s)) return -1;
            H *= 2; W *= 2;
            if (f.conv("decoder.up_blocks." + std::to_string(i) + ".upsamplers.0.conv", T, H, W, Y, nullptr)) return -1;
            ix = (ix + 3) & 3;
        }
    }
    float* X = d->buf[ix];
    float* T = d->buf[(ix + 1) & 3];
    float* Y = d->buf[(ix + 3) & 3];
    if (f.gn("decoder.conv_norm_out", X, T, H, W, 1, 0)) return -1;
    if (f.conv("decoder.conv_out", T, H, W, Y, nullptr)) return -1;
    return padded_to_nchw(Y, out_nchw, B, c.out_channels, round32(c.out_channels), H, W, s);
}

MMDP_API int mmdp_vqmodel_encode(mmdp_vqdec* d, const float* pixels_nchw, int B, int H, int W, float* latents_nchw, void* stream) {
    if (!d || !pixels_nchw || !latents_nchw) return set_error("mmdp_vqmodel_encode: null argument");
    if (!d->is_vqmodel) return set_error("mmdp_vqmodel_encode: not a VQModel context (create it with mmdp_vqmodel_create)");
    const mmdp_vqmodel_config& c = d->vm;
    const int L = c.n_levels, smax = 1 << (L - 1);
    if (H < smax || W < smax || H % smax || W % smax)
        return set_error("mmdp_vqmodel_encode: %dx%d pixels are not a positive multiple of the downscale %d", H, W, smax);
    if (vqmodel_check(d, "mmdp_vqmodel_encode", B, H / smax, W / smax)) return -1;
    cudaStream_t s = (cudaStream_t)stream;
    Fwd f{d, s, B};
    if (nchw_to_padded(pixels_nchw, d->buf[0], B, c.in_channels, round32(c.in_channels), H, W, s)) return -1;
    if (f.conv("encoder.conv_in", d->buf[0], H, W, d->buf[1], nullptr)) return -1;
    int ix = 1;
    for (int i = 0; i < L; ++i) {
        for (int j = 0; j < c.layers_per_block; ++j)
            if (f.resblock(blk("encoder.down_blocks.", i, ".resnets.", j), H, W, ix)) return -1;
        if (i != L - 1) {
            // Downsample2D with padding 0: F.pad (0, 1, 0, 1) + 3x3 stride-2 convolution (see downsample_pick)
            const int C = c.block_out_channels[i];
            float* X = d->buf[ix];
            float* T = d->buf[(ix + 1) & 3];
            float* Y = d->buf[(ix + 3) & 3];
            if (f.conv("encoder.down_blocks." + std::to_string(i) + ".downsamplers.0.conv", X, H, W, T, nullptr)) return -1;
            if (downsample_pick(T, Y, B, C, H, W, s)) return -1;
            H /= 2; W /= 2;
            ix = (ix + 3) & 3;
        }
    }
    if (mid_block(f, "encoder.mid_block", H, W, ix, c.mid_block_add_attention != 0)) return -1;
    float* X = d->buf[ix];
    float* T = d->buf[(ix + 1) & 3];
    float* Y = d->buf[(ix + 3) & 3];
    if (f.gn("encoder.conv_norm_out", X, T, H, W, 1, 0)) return -1;
    const int zc = round32(c.latent_channels);
    MMDP_CUDA(cudaMemsetAsync(Y, 0, (size_t)B * (H + 2) * (W + 2) * zc * 4, s));  // channels lat..zc stay zero (quant_conv input)
    if (f.conv("encoder.conv_out", T, H, W, Y, nullptr)) return -1;
    if (f.conv("quant_conv", Y, H, W, X, nullptr)) return -1;
    return padded_to_nchw(X, latents_nchw, B, c.latent_channels, zc, H, W, s);
}

MMDP_API int mmdp_vqmodel_error_flags(mmdp_vqdec* d, int32_t* flags_host, void* stream) {
    if (!d || !flags_host) return set_error("mmdp_vqmodel_error_flags: null argument");
    if (!d->is_vqmodel) return set_error("mmdp_vqmodel_error_flags: not a VQModel context");
    cudaStream_t s = (cudaStream_t)stream;
    int v = 0;
    MMDP_CUDA(cudaMemcpyAsync(&v, d->err, sizeof(int), cudaMemcpyDeviceToHost, s));
    MMDP_CUDA(cudaMemsetAsync(d->err, 0, sizeof(int), s));
    MMDP_CUDA(cudaStreamSynchronize(s));
    *flags_host = v;
    return 0;
}

}  // extern "C"
