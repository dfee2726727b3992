// Host runtime helpers: error reporting, device properties, TMA tensor-map construction.
// libcuda is NOT linked: cuTensorMapEncodeTiled is resolved through cudaGetDriverEntryPoint so the
// library loads (and exports its symbols) on a CPU-only box; calling into it without a GPU fails loudly.
#include "mmdp_internal.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>
#include <vector>

namespace mmdp {

static thread_local char g_err[1024] = "";

int set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return -1;
}
const char* last_error() { return g_err; }

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 132;
        n = prop.multiProcessorCount;
    }
    return n;
}

int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return (e && *e) ? atoi(e) : dflt;
}

// Tuning options: initialised from the environment on first use, changeable at run time with mmdp_set_option().
struct Opt { const char* key; const char* env; int dflt; int val; bool init; };
static Opt g_opts[OPT_COUNT] = {
    {"pdl", "MMDP_PDL", 1, 0, false},
    {"gemm_splitk", "MMDP_GEMM_SPLITK", 2, 0, false},
    {"gemm_l2pf", "MMDP_GEMM_L2PF", 0, 0, false},
    {"gemm_l2pf_mod", "MMDP_GEMM_L2PF_MOD", 4, 0, false},
    {"gemm_group_m", "MMDP_GEMM_GROUP_M", -1, 0, false},
    {"attn_split_tail", "MMDP_ATTN_SPLIT_TAIL", 1, 0, false},
    {"rmsnorm_warp", "MMDP_RMSNORM_WARP", 1, 0, false},
    {"row_window", "MMDP_ROW_WINDOW", 1, 0, false},
    {"attn_version", "MMDP_ATTN_VERSION", 6, 0, false},
    {"gemm_pair", "MMDP_GEMM_PAIR", 0, 0, false},  // pairs measured slower on an H100 (gemm.cu)
};
int opt(int id) {
    Opt& o = g_opts[id];
    if (!o.init) { o.val = env_int(o.env, o.dflt); o.init = true; }
    return o.val;
}
int set_opt(const char* key, int value) {
    for (int i = 0; i < OPT_COUNT; ++i)
        if (!strcmp(g_opts[i].key, key)) { g_opts[i].val = value; g_opts[i].init = true; return 0; }
    return set_error("mmdp_set_option: unknown option '%s'", key);
}
int pdl_mode() { return opt(OPT_PDL) ? 1 : 0; }
void set_pdl_mode(int on) { set_opt("pdl", on ? 1 : 0); }

// ------------------------------------------------------------------------------------------------
// launch accounting / profiling
// ------------------------------------------------------------------------------------------------
struct ProfRec { cudaEvent_t e0, e1; int kind; double work; };
static std::vector<ProfRec> g_prof;
static size_t g_prof_used = 0;
static bool g_prof_on = false;
static long long g_launches = 0;

LaunchScope::LaunchScope(int kind, double work, cudaStream_t s) : idx(-1), stream(s) {
    ++g_launches;
    if (!g_prof_on) return;
    if (g_prof_used == g_prof.size()) {
        ProfRec r{};
        if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
        g_prof.push_back(r);
    }
    idx = (int)g_prof_used++;
    g_prof[idx].kind = kind;
    g_prof[idx].work = work;
    cudaEventRecord(g_prof[idx].e0, s);
}
LaunchScope::~LaunchScope() {
    if (idx >= 0) cudaEventRecord(g_prof[idx].e1, stream);
}
void prof_enable(int on) {
    g_prof_on = on != 0;
    g_prof_used = 0;
}
int prof_summary(double* ms, double* work, long long* launches) {
    MMDP_CUDA(cudaDeviceSynchronize());
    for (int k = 0; k < LK_COUNT; ++k) { ms[k] = 0; work[k] = 0; launches[k] = 0; }
    for (size_t i = 0; i < g_prof_used; ++i) {
        float t = 0.f;
        MMDP_CUDA(cudaEventElapsedTime(&t, g_prof[i].e0, g_prof[i].e1));
        ms[g_prof[i].kind] += t;
        work[g_prof[i].kind] += g_prof[i].work;
        launches[g_prof[i].kind] += 1;
    }
    return 0;
}
long long launch_count(int reset) {
    long long v = g_launches;
    if (reset) g_launches = 0;
    return v;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                      uint32_t box_cols) {
    return make_tmap_2d(out, base, 2, rows, cols, ld, box_rows, box_cols);
}

// Encoded tensor maps are cached per (base, shape, stride, box): a forward re-uses the same ~10 buffers x ~130 weight
// matrices on every call, and cuTensorMapEncodeTiled costs ~1-2 us of host time per call (2-3 per GEMM / attention launch).
struct TmapKey {
    const void* base;
    uint64_t rows, cols, ld;
    uint32_t box_rows, box_cols;
    int elem_bytes;
    bool operator==(const TmapKey& o) const {
        return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
               box_cols == o.box_cols && elem_bytes == o.elem_bytes;
    }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        uint64_t h = reinterpret_cast<uint64_t>(k.base) * 0x9E3779B97F4A7C15ull;
        h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
        h ^= (k.cols * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2));
        h ^= (k.ld + ((uint64_t)k.box_rows << 32) + ((uint64_t)k.box_cols << 8) + (uint64_t)k.elem_bytes + (h << 6) + (h >> 2));
        return (size_t)h;
    }
};
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmaps;
static std::mutex g_tmap_mu;

int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return set_error("cuTensorMapEncodeTiled not available (no CUDA driver / no GPU)");
    if (elem_bytes != 2 && elem_bytes != 4) return set_error("tmap: element size must be 2 (bf16) or 4 (fp32)");
    if (box_cols * (uint32_t)elem_bytes != 128) return set_error("tmap: box must be exactly one 128-byte swizzle atom wide");
    if (box_rows == 0 || box_rows > 256) return set_error("tmap: box_rows out of range");
    const TmapKey key{base, rows, cols, ld, box_rows, box_cols, elem_bytes};
    {
        std::lock_guard<std::mutex> lk(g_tmap_mu);
        auto it = g_tmaps.find(key);
        if (it != g_tmaps.end()) {
            *out = it->second;
            return 0;
        }
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld * (uint64_t)elem_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error("cuTensorMapEncodeTiled failed (%d) base=%p rows=%llu cols=%llu ld=%llu box=[%u,%u]", (int)r,
                         base, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows,
                         box_cols);
    {
        std::lock_guard<std::mutex> lk(g_tmap_mu);
        if (g_tmaps.size() >= 8192) g_tmaps.clear();  // bounded: callers with ever-changing buffers just re-encode
        g_tmaps.emplace(key, *out);
    }
    return 0;
}

}  // namespace mmdp
