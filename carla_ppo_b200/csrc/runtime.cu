// Library runtime behind the C ABI: the error buffer, the launch counter, the per-call-site profiler, the math mode, the
// per-device kernel setup, the tensor-core debug entry points and Adam (which both VAEs' train steps call).
#include <mutex>
#include <stdarg.h>

#include "vae_shared.cuh"

namespace cpb {

static thread_local char g_err[512] = "";
int64_t g_launches = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---- profiling -------------------------------------------------------------------------------
bool g_profile_on = false;
namespace {
struct ProfRec { const char* label; cudaEvent_t a, b; };
constexpr int kMaxProfRecs = 4096;
ProfRec g_recs[kMaxProfRecs];
int g_nrecs = 0;
int g_open = -1;
}
void profile_begin(const char* label, cudaStream_t s) {
    if (g_nrecs >= kMaxProfRecs) { g_open = -1; return; }
    ProfRec& r = g_recs[g_nrecs];
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) { g_open = -1; return; }
    r.label = label;
    cudaEventRecord(r.a, s);
    g_open = g_nrecs++;
}
void profile_end(cudaStream_t s) {
    if (g_open >= 0) cudaEventRecord(g_recs[g_open].b, s);
    g_open = -1;
}

// 0: fp32 SIMT everywhere; 1: 3xTF32 wgmma for the dense conv/deconv layers; 2: the same layers as ONE TF32 wgmma
// pass with operands rounded to nearest (not fp32-accurate: up to 2^-10 relative error per product)
int g_math_mode = 1;
int tc_passes() { return g_math_mode == 2 ? 1 : 3; }
// Per-device one-time setup (cudaFuncSetAttribute for > 48 KB dynamic shared memory and the co-resident cluster counts
// of the persistent kernels are PER DEVICE): keyed by cudaGetDevice() so that a process driving several GPUs works.
constexpr int kMaxDevices = 64;
static std::mutex g_init_mutex;
static int g_init_done[kMaxDevices];     // 0: not yet, 1: ok, 2: failed
static int32_t g_init_status[kMaxDevices];
int32_t ensure_init() {
    int dev = 0;
    CPB_CUDA(cudaGetDevice(&dev));
    CPB_REQUIRE(dev >= 0 && dev < kMaxDevices, "device ordinal %d out of range", dev);
    std::lock_guard<std::mutex> lock(g_init_mutex);
    if (g_init_done[dev] == 0) {
        int32_t st = tapgemm_init();
        if (st == CPB_OK) st = wgrad_init();
        if (st == CPB_OK) st = edge_init();
        if (st == CPB_OK) st = tc_tapgemm_init();
        if (st == CPB_OK) st = tc_wgrad_init();
        g_init_status[dev] = st;
        g_init_done[dev] = st == CPB_OK ? 1 : 2;
    }
    return g_init_status[dev];
}

// CPB_TC_DEBUG: timing decomposition of the tensor-core kernels (results are wrong when set; see tapgemm.cuh)
int tc_debug_flags() {
    static const int v = [] { const char* e = getenv("CPB_TC_DEBUG"); return e ? atoi(e) : 0; }();
    return v;
}

}  // namespace cpb

using namespace cpb;

extern "C" {

const char* cpb_last_error(void) { return cpb::g_err; }
const char* cpb_build_info(void) { return "carla_ppo_b200 0.3 (sm_90a; wgmma 3xTF32 + fp32 SIMT tap-GEMM)"; }
int64_t cpb_launch_count(void) { return cpb::g_launches; }
void cpb_reset_launch_count(void) { cpb::g_launches = 0; }

/* debug: D[M,N] = A[M,K] * Bt[N,K]^T through the tensor-core tap-GEMM (dense, one tap); the single-pass kernel in math
   mode 2, 3xTF32 otherwise.  scratch: at least 2*N*K floats (the weight image); callers sized for an older layout pass
   2*N*K + M*K, of which the rest goes unused. */
int32_t cpb_debug_tc_gemm(const float* a, const float* bt, float* d, int32_t m, int32_t n, int32_t k, float* scratch, void* stream) {
    CPB_TRY(ensure_init());
    cudaStream_t s = (cudaStream_t)stream;
    TcWeightTable w;
    memset(&w, 0, sizeof(w));
    w.njobs = 1; w.total = (long long)n * k;
    w.jobs[0].src_off = 0; w.jobs[0].dst_hi = 0; w.jobs[0].dst_lo = (long long)n * k; w.jobs[0].mode = 0; w.jobs[0].N = n; w.jobs[0].C = k; w.jobs[0].count = w.total;
    w.jobs[0].round_nearest = tc_passes() == 1 ? 1 : 0;
    TapGemmParams p = dense_problem(a, m, k, nullptr, n, nullptr, nullptr, d, 0);
    p.wk_hi = scratch; p.wk_lo = scratch + (long long)n * k;
    p.debug = tc_debug_flags();
    p.passes = tc_passes();
    CPB_TRY(launch_tc_weights(bt, scratch, w, s));
    return launch_tc_tapgemm(p, s);
}

/* debug: out[I,J] = big[M,I]^T small[M,J] through the tensor-core wgrad kernel (1x1 "image", one tap); the single-pass
   kernel in math mode 2, 3xTF32 otherwise. */
int32_t cpb_debug_tc_wgrad(const float* big, const float* small, float* out, int32_t m, int32_t i, int32_t j,
                           int32_t variant, float* partial, void* stream) {
    CPB_TRY(ensure_init());
    cudaStream_t s = (cudaStream_t)stream;
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = big; w.small = small; w.partial = partial;
    w.batch = m; w.Wb = 1; w.big_pitch = i; w.big_img = i; w.Ho = w.Wo = 1; w.sstride = 1;
    w.ntaps = 1; w.run = i; w.tap_off[0] = 0; w.I = i; w.J = j; w.tc_variant = variant;
    w.passes = tc_passes();
    w.splits = 2;
    w.m_per_split = align_up(((long long)m + 1) / 2, 32);
    CPB_TRY(launch_tc_wgrad(w, s));
    return launch_reduce_partials(partial, w.splits, i, j, i, i, j, out, s);
}

int32_t cpb_set_math_mode(int32_t mode) {
    CPB_REQUIRE(mode >= 0 && mode <= 2, "math mode must be 0 (fp32 SIMT), 1 (3xTF32 wgmma) or 2 (single-pass TF32 wgmma), got %d", mode);
    cpb::g_math_mode = mode;
    return CPB_OK;
}
int32_t cpb_get_math_mode(void) { return cpb::g_math_mode; }

void cpb_profile_enable(int32_t on) { cpb::g_profile_on = on != 0; }
void cpb_profile_reset(void) {
    for (int i = 0; i < cpb::g_nrecs; ++i) { cudaEventDestroy(cpb::g_recs[i].a); cudaEventDestroy(cpb::g_recs[i].b); }
    cpb::g_nrecs = 0;
    cpb::g_open = -1;
}
int64_t cpb_profile_report(char* buf, int64_t capacity) {
    cudaDeviceSynchronize();
    struct Agg { const char* label; int count; double ms; };
    static Agg agg[256];
    int nagg = 0;
    for (int i = 0; i < cpb::g_nrecs; ++i) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, cpb::g_recs[i].a, cpb::g_recs[i].b) != cudaSuccess) continue;
        int j = 0;
        for (; j < nagg; ++j) if (strcmp(agg[j].label, cpb::g_recs[i].label) == 0) break;
        if (j == nagg) { if (nagg == 256) continue; agg[nagg++] = Agg{cpb::g_recs[i].label, 0, 0.0}; }
        agg[j].count++; agg[j].ms += ms;
    }
    int64_t off = 0;
    for (int j = 0; j < nagg; ++j) {
        int n = snprintf(buf + off, capacity > off ? (size_t)(capacity - off) : 0, "%s %d %.6f\n", agg[j].label, agg[j].count, agg[j].ms);
        if (n < 0 || off + n >= capacity) break;
        off += n;
    }
    return off;
}

int32_t cpb_adam_apply(float* params, const float* grads, float* m, float* v, int64_t n, float* powers, float lr,
                       const float* lr_dev, float beta1, float beta2, float epsilon, void* stream) {
    CPB_REQUIRE(params && grads && m && v && powers, "adam: NULL pointer");
    ProfScope prof("adam", (cudaStream_t)stream);
    return launch_adam(params, grads, m, v, n, powers, lr, lr_dev, beta1, beta2, epsilon, (cudaStream_t)stream);
}

int32_t cpb_adam_apply_guarded(float* params, const float* grads, float* m, float* v, int64_t n, float* powers, float lr,
                               const float* lr_dev, float beta1, float beta2, float epsilon, const void* guard, void* stream) {
    CPB_REQUIRE(params && grads && m && v && powers, "adam: NULL pointer");
    ProfScope prof("adam", (cudaStream_t)stream);
    return launch_adam(params, grads, m, v, n, powers, lr, lr_dev, beta1, beta2, epsilon, (cudaStream_t)stream, guard);
}

}  // extern "C"
