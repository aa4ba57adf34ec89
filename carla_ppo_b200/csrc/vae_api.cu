// ConvVAE orchestration behind the C ABI (include/carla_ppo_b200.h).
// Replaces the TF graph built by reference vae/models.py:85-142 + 249-266 and the sess.run calls of
// VAE.encode / generate_from_latent / reconstruct / evaluate / train_one_epoch (:188-231).
#include <algorithm>
#include <mutex>
#include <stdarg.h>

#include "elementwise.cuh"
#include "tapgemm.cuh"
#include "wgrad.cuh"

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

int g_math_mode = 1;   // 0: fp32 SIMT everywhere; 1: 3xTF32 wgmma for the dense conv/deconv layers
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
        if (st == CPB_OK) st = tc_tapgemm_init();
        if (st == CPB_OK) st = tc_wgrad_init();
        g_init_status[dev] = st;
        g_init_done[dev] = st == CPB_OK ? 1 : 2;
    }
    return g_init_status[dev];
}

// ---------------------------------------------------------------------------------------------
// geometry (source 80x160x3, reference vae_common.py:18-20; layer table SURVEY appendix A.1)
// ---------------------------------------------------------------------------------------------
namespace geo {
constexpr int H0 = 80, W0 = 160;
constexpr int H1 = 39, W1 = 79, C1 = 32;
constexpr int H2 = 18, W2 = 38, C2 = 64;
constexpr int H3 = 8, W3 = 18, C3 = 128;
constexpr int H4 = 3, W4 = 8, C4 = 256;
constexpr int FEAT = H4 * W4 * C4;   // 6144
constexpr int NPIX = H0 * W0;        // 12800
}  // namespace geo

enum VaeTensor {
    T_CONV1_K, T_CONV1_B, T_CONV2_K, T_CONV2_B, T_CONV3_K, T_CONV3_B, T_CONV4_K, T_CONV4_B,
    T_MEAN_K, T_MEAN_B, T_LOGVAR_K, T_LOGVAR_B, T_DENSE1_K, T_DENSE1_B,
    T_DECONV1_K, T_DECONV1_B, T_DECONV2_K, T_DECONV2_B, T_DECONV3_K, T_DECONV3_B, T_DECONV4_K, T_DECONV4_B,
    T_COUNT
};

static const char* kVaeNames[T_COUNT] = {
    "encoder/conv1/kernel", "encoder/conv1/bias", "encoder/conv2/kernel", "encoder/conv2/bias",
    "encoder/conv3/kernel", "encoder/conv3/bias", "encoder/conv4/kernel", "encoder/conv4/bias",
    "mean/kernel", "mean/bias", "logstd_sqare/kernel", "logstd_sqare/bias",
    "decoder/dense1/kernel", "decoder/dense1/bias",
    "decoder/deconv1/kernel", "decoder/deconv1/bias", "decoder/deconv2/kernel", "decoder/deconv2/bias",
    "decoder/deconv3/kernel", "decoder/deconv3/bias", "decoder/deconv4/kernel", "decoder/deconv4/bias"};

struct VaeLayout {
    int64_t off[T_COUNT];
    int64_t size[T_COUNT];
    int32_t shape[T_COUNT][4];
    int64_t total;
};

static void set_shape(VaeLayout& L, int t, int a, int b = 0, int c = 0, int d = 0) {
    L.shape[t][0] = a; L.shape[t][1] = b; L.shape[t][2] = c; L.shape[t][3] = d;
    int64_t n = a;
    if (b) n *= b;
    if (c) n *= c;
    if (d) n *= d;
    L.size[t] = n;
}

static VaeLayout make_layout(int ct, int z) {
    using namespace geo;
    VaeLayout L;
    set_shape(L, T_CONV1_K, 4, 4, 3, C1);    set_shape(L, T_CONV1_B, C1);
    set_shape(L, T_CONV2_K, 4, 4, C1, C2);   set_shape(L, T_CONV2_B, C2);
    set_shape(L, T_CONV3_K, 4, 4, C2, C3);   set_shape(L, T_CONV3_B, C3);
    set_shape(L, T_CONV4_K, 4, 4, C3, C4);   set_shape(L, T_CONV4_B, C4);
    set_shape(L, T_MEAN_K, FEAT, z);         set_shape(L, T_MEAN_B, z);
    set_shape(L, T_LOGVAR_K, FEAT, z);       set_shape(L, T_LOGVAR_B, z);
    set_shape(L, T_DENSE1_K, z, FEAT);       set_shape(L, T_DENSE1_B, FEAT);
    set_shape(L, T_DECONV1_K, 4, 4, C3, C4); set_shape(L, T_DECONV1_B, C3);
    set_shape(L, T_DECONV2_K, 4, 4, C2, C3); set_shape(L, T_DECONV2_B, C2);
    set_shape(L, T_DECONV3_K, 5, 5, C1, C2); set_shape(L, T_DECONV3_B, C1);
    set_shape(L, T_DECONV4_K, 4, 4, ct, C1); set_shape(L, T_DECONV4_B, ct);
    // storage order: TF creation order, except that the two head kernels (and the two head biases) are
    // adjacent so that both heads run as one y-batched tap-GEMM.
    static const int order[T_COUNT] = {
        T_CONV1_K, T_CONV1_B, T_CONV2_K, T_CONV2_B, T_CONV3_K, T_CONV3_B, T_CONV4_K, T_CONV4_B,
        T_MEAN_K, T_LOGVAR_K, T_MEAN_B, T_LOGVAR_B, T_DENSE1_K, T_DENSE1_B,
        T_DECONV1_K, T_DECONV1_B, T_DECONV2_K, T_DECONV2_B, T_DECONV3_K, T_DECONV3_B, T_DECONV4_K, T_DECONV4_B};
    int64_t o = 0;
    for (int i = 0; i < T_COUNT; ++i) {
        L.off[order[i]] = o;
        o += align_up(L.size[order[i]], 64);
    }
    L.total = o;
    return L;
}

// ---------------------------------------------------------------------------------------------
// workspace plan
// ---------------------------------------------------------------------------------------------
struct TcW { int64_t f_hi, f_lo, t_hi, t_lo; };   // gather-form / quad-scatter-form K-major hi/lo copies of one kernel
struct Relayout {
    int64_t conv2T, conv3T, conv4T, deconv1T, deconv2T, deconv3T, dense1T, headsT, conv1P, deconv4P;
    TcW tc[6];          // conv2, conv3, conv4, deconv1, deconv2, deconv3
    int64_t total;
};
enum { TC_CONV2, TC_CONV3, TC_CONV4, TC_DECONV1, TC_DECONV2, TC_DECONV3 };

static Relayout make_relayout(int z) {
    using namespace geo;
    Relayout r;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
    r.conv2T = take(16LL * C1 * C2);
    r.conv3T = take(16LL * C2 * C3);
    r.conv4T = take(16LL * C3 * C4);
    r.deconv1T = take(16LL * C3 * C4);
    r.deconv2T = take(16LL * C2 * C3);
    r.deconv3T = take(25LL * C1 * C2);
    r.dense1T = take((int64_t)z * FEAT);
    r.headsT = take(2LL * z * FEAT);
    r.conv1P = take(16LL * 4 * C1);
    r.deconv4P = take(16LL * 4 * C1);
    const int64_t sizes[6] = {16LL * C1 * C2, 16LL * C2 * C3, 16LL * C3 * C4, 16LL * C3 * C4, 16LL * C2 * C3, 25LL * C1 * C2};
    const int64_t qsizes[6] = {16LL * C1 * C2, 16LL * C2 * C3, 16LL * C3 * C4, 16LL * C3 * C4, 16LL * C2 * C3, 36LL * C1 * C2};
    for (int i = 0; i < 6; ++i) {
        r.tc[i].f_hi = take(sizes[i]); r.tc[i].f_lo = take(sizes[i]);
        r.tc[i].t_hi = take(qsizes[i]); r.tc[i].t_lo = take(qsizes[i]);
    }
    r.total = o;
    return r;
}

struct VaePlan {
    int B, ct, z, mode;
    Relayout rl;
    float *relayout, *xp, *yp, *a1, *a2, *a3, *a4, *heads, *zbuf, *kl_rows, *kl_active, *frame_loss;
    float *d1, *b1, *b2, *b3, *logits_p;
    float *gA, *gB, *gz, *gheads, *partial, *colsum;
    float* cs_edge;     // per-CTA column sums of deconv4's data gradient (edge_gather), [edge_gather_blocks(B)][32]
    float* frame_dsum;  // per-frame channel sums of d loss / d logits, [B][4]
    float* lo;          // lo plane scratch for tensor-core sources whose producer does not write one (small tensors)
    float *a1_lo, *a2_lo, *a3_lo, *b1_lo, *b2_lo, *gA_lo, *gB_lo;   // lo planes written by the producing kernels
    float* ksplit;      // partial results of the k-split dense layers: kMaxKSplit x [2, B, z]
    int64_t bytes;
    bool ok;
};

static int64_t max_partial_floats(int B, int z) {
    using namespace geo;
    struct P { int I, J; long long M; };
    const P ps[] = {
        {64, C1, (long long)B * H1 * W1},          // conv1 / deconv4 (padded to 4 channels)
        {16 * C1, C2, (long long)B * H2 * W2},     // conv2
        {16 * C2, C3, (long long)B * H3 * W3},     // conv3 / deconv2
        {16 * C3, C4, (long long)B * H4 * W4},     // conv4 / deconv1
        {25 * C1, C2, (long long)B * H2 * W2},     // deconv3
        {FEAT, z, (long long)B},                    // heads
        {z, FEAT, (long long)B},                    // dense1
    };
    int64_t best = (int64_t)edge_wgrad_ctas(B) * 48 * C1;
    // the tensor-core weight gradient runs ONE wave of (i-tile, j-tile, split) CTAs with 128 x BN <= 128 x 64 tiles
    if (best < (int64_t)kTcWaveCtas * 128 * 64) best = (int64_t)kTcWaveCtas * 128 * 64;
    for (const P& p : ps) {
        int64_t n = (int64_t)wgrad_pick_splits(p.I, p.J, p.M) * p.I * p.J;
        if (n > best) best = n;
        n = (int64_t)tc_wgrad_pick_splits(p.I, p.J, p.M) * p.I * p.J;
        if (n > best) best = n;
    }
    return best;
}

static VaePlan make_plan(void* ws, int64_t ws_bytes, int B, int ct, int z, int mode) {
    using namespace geo;
    VaePlan p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.ct = ct; p.z = z; p.mode = mode;
    p.rl = make_relayout(z);
    Arena a(ws, ws_bytes);
    const int64_t b = B;
    p.relayout = a.take<float>(p.rl.total);
    p.xp = a.take<float>(b * NPIX * 4);
    p.a1 = a.take<float>(b * H1 * W1 * C1);
    p.a2 = a.take<float>(b * H2 * W2 * C2);
    p.a3 = a.take<float>(b * H3 * W3 * C3);
    p.a4 = a.take<float>(b * FEAT);
    p.heads = a.take<float>(2 * b * z);
    p.lo = a.take<float>(b * FEAT);
    p.ksplit = a.take<float>((int64_t)kMaxKSplit * 2 * b * z);
    // lo planes (x - trunc_tf32(x)): the second TF32 operand of every tensor-core source, written by its producer
    p.a1_lo = a.take<float>(b * H1 * W1 * C1);
    p.a2_lo = a.take<float>(b * H2 * W2 * C2);
    p.a3_lo = a.take<float>(b * H3 * W3 * C3);
    if (mode >= CPB_WS_FORWARD) {
        p.yp = a.take<float>(b * NPIX * 4);
        p.zbuf = a.take<float>(b * z);
        p.kl_rows = a.take<float>(b);
        p.kl_active = a.take<float>(b);
        p.frame_loss = a.take<float>(b);
        p.d1 = a.take<float>(b * FEAT);
        p.b1 = a.take<float>(b * H3 * W3 * C3);
        p.b1_lo = a.take<float>(b * H3 * W3 * C3);
        p.b2_lo = a.take<float>(b * H2 * W2 * C2);
        p.b2 = a.take<float>(b * H2 * W2 * C2);
        p.b3 = a.take<float>(b * H1 * W1 * C1);
        p.logits_p = a.take<float>(b * NPIX * 4);
    }
    if (mode >= CPB_WS_TRAIN) {
        p.gA = a.take<float>(b * H1 * W1 * C1);
        p.gB = a.take<float>(b * H1 * W1 * C1);
        p.gA_lo = a.take<float>(b * H1 * W1 * C1);
        p.gB_lo = a.take<float>(b * H1 * W1 * C1);
        p.gz = a.take<float>(b * z);
        p.gheads = a.take<float>(2 * b * z);
        p.partial = a.take<float>(max_partial_floats(B, z));
        p.colsum = a.take<float>(colsum_scratch_floats(b * NPIX, 4) + colsum_scratch_floats(b * H1 * W1, C1) +
                                 colsum_scratch_floats(b, FEAT));
        p.cs_edge = a.take<float>(edge_gather_blocks(B) * C1);
        p.frame_dsum = a.take<float>(b * 4);
    }
    p.bytes = a.off;
    p.ok = ws == nullptr || !a.overflow;
    return p;
}

// ---------------------------------------------------------------------------------------------
// tap-GEMM problem builders
// ---------------------------------------------------------------------------------------------
static TapGemmParams base_params() {
    TapGemmParams p;
    memset(&p, 0, sizeof(p));
    p.nclass = 1;
    p.ybatch = 1;
    p.ksplit = 1;
    return p;
}

// gather form: small[b,i,j,:] = sum_{kh,kw,cb} big[b,2i+kh,2j+kw,cb] * W[kh,kw,cb,:]
static TapGemmParams gather_problem(const float* big, int B, int Hb, int Wb, int pitch, int k, const float* W,
                                    int N, const float* bias, const float* mask, float* small, int relu,
                                    const float* wk_hi = nullptr, const float* wk_lo = nullptr) {
    TapGemmParams p = base_params();
    p.wk_hi = wk_hi; p.wk_lo = wk_lo;
    p.src = big; p.wmat = W; p.bias = bias; p.mask = mask; p.dst = small;
    p.batch = B; p.Hs = Hb; p.Ws = Wb; p.src_pitch = pitch; p.src_img = (long long)Hb * Wb * pitch;
    p.sstride = 2; p.C = k * pitch; p.N = N; p.ldw = N;
    const int Ho = (Hb - k) / 2 + 1, Wo = (Wb - k) / 2 + 1;
    p.Hd = Ho; p.Wd = Wo; p.dstride = 1; p.dst_pitch = N; p.dst_img = (long long)Ho * Wo * N;
    p.relu = relu; p.check = 0;
    TapClass& c = p.cls[0];
    c.ntaps = k; c.py = c.px = 0; c.Ho = Ho; c.Wo = Wo;
    for (int kh = 0; kh < k; ++kh) {
        c.taps[kh].dy = kh; c.taps[kh].dx = 0;
        c.taps[kh].src_off = (long long)kh * Wb * pitch;
        c.taps[kh].w_off = (long long)kh * k * pitch * N;
    }
    return p;
}

// scatter form: big[b,2i+kh,2j+kw,cb] += small[b,i,j,cs] * W[kh,kw,cb,cs]; Wt is [kh][kw][cs][cb]
static TapGemmParams scatter_problem(const float* small, int B, int Hs, int Ws, int Cs, int k, const float* Wt,
                                     int Cb, const float* bias, const float* mask, float* big, int Hb, int Wb,
                                     int relu, const float* wk_hi = nullptr, const float* wk_lo = nullptr) {
    TapGemmParams p = base_params();
    p.wk_hi = wk_hi; p.wk_lo = wk_lo;
    p.src = small; p.wmat = Wt; p.bias = bias; p.mask = mask; p.dst = big;
    p.batch = B; p.Hs = Hs; p.Ws = Ws; p.src_pitch = Cs; p.src_img = (long long)Hs * Ws * Cs;
    p.sstride = 1; p.C = Cs; p.N = Cb; p.ldw = Cb;
    p.Hd = Hb; p.Wd = Wb; p.dstride = 2; p.dst_pitch = Cb; p.dst_img = (long long)Hb * Wb * Cb;
    p.relu = relu; p.check = 1; p.nclass = 4;
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            TapClass& c = p.cls[py * 2 + px];
            c.py = py; c.px = px;
            c.Ho = (Hb - py + 1) / 2; c.Wo = (Wb - px + 1) / 2;
            int n = 0;
            for (int kh = py, j = 0; kh < k; kh += 2, ++j)
                for (int kw = px, i = 0; kw < k; kw += 2, ++i) {
                    Tap& t = c.taps[n++];
                    t.dy = -j; t.dx = -i;
                    t.src_off = ((long long)(-j) * Ws - i) * Cs;
                    t.w_off = ((long long)kh * k + kw) * Cs * Cb;
                }
            c.ntaps = n;
        }
    return p;
}

// dense: dst[b, :N] = src[b, :K] @ W[K, ldw] (+bias)
static TapGemmParams dense_problem(const float* src, int B, int K, const float* W, int N, const float* bias,
                                   const float* mask, float* dst, int relu) {
    TapGemmParams p = base_params();
    p.src = src; p.wmat = W; p.bias = bias; p.mask = mask; p.dst = dst;
    p.batch = B; p.Hs = p.Ws = 1; p.src_pitch = K; p.src_img = K; p.sstride = 1; p.C = K; p.N = N; p.ldw = N;
    p.Hd = p.Wd = 1; p.dstride = 1; p.dst_pitch = N; p.dst_img = N; p.relu = relu; p.check = 0;
    TapClass& c = p.cls[0];
    c.ntaps = 1; c.py = c.px = 0; c.Ho = c.Wo = 1;
    c.taps[0].dy = c.taps[0].dx = 0; c.taps[0].src_off = 0; c.taps[0].w_off = 0;
    return p;
}

// Re-express a 4-class scatter-form problem as ONE quad-fused GEMM (tensor-core path): rows = 2x2 output quads,
// columns = (class, cb), taps = the union window; needs the mode-2 weights of tc_weights_kernel.
static TapGemmParams quad_from_scatter(const TapGemmParams& sp, int k) {
    TapGemmParams p = sp;
    const int Cb = sp.N, Cs = sp.C;
    p.quad = 1; p.quad_cb = Cb; p.N = 4 * Cb; p.nclass = 1; p.check = 1;
    TapClass& c = p.cls[0];
    const int win = (k + 1) / 2;
    c.py = c.px = 0;
    c.Ho = (sp.Hd + 1) / 2; c.Wo = (sp.Wd + 1) / 2;
    c.ntaps = win * win;
    for (int j = 0; j < win; ++j)
        for (int i = 0; i < win; ++i) {
            Tap& t = c.taps[j * win + i];
            t.dy = -j; t.dx = -i;
            t.src_off = ((long long)(-j) * sp.Ws - i) * Cs;
            t.w_off = (long long)(j * win + i) * 4 * Cb * Cs;
        }
    return p;
}

// CPB_TC_DEBUG: timing decomposition of the tensor-core kernels (results are wrong when set; see tapgemm.cuh)
static int tc_debug_flags() {
    static const int v = [] { const char* e = getenv("CPB_TC_DEBUG"); return e ? atoi(e) : 0; }();
    return v;
}

static thread_local float* tl_lo_scratch = nullptr;   // lo plane of the current tensor-core source (VaePlan::lo)

// src_lo / dst_lo: lo planes (x - trunc_tf32(x)) of the source (written by its producer; nullptr: computed here into the
// scratch plane) and of the destination (written by the epilogue for the consuming layer; nullptr: not needed)
static int32_t tg(const char* label, const TapGemmParams& p, cudaStream_t s, int scatter_k = 0,
                  const float* src_lo = nullptr, float* dst_lo = nullptr) {
    ProfScope prof(label, s);
    if (g_math_mode == 1 && p.wk_hi != nullptr && tl_lo_scratch != nullptr) {
        TapGemmParams q = scatter_k > 0 ? quad_from_scatter(p, scatter_k) : p;
        q.debug = tc_debug_flags();
        q.src_lo = src_lo != nullptr ? src_lo : tl_lo_scratch;
        q.dst_lo = dst_lo;
        if (tc_tapgemm_supported(q)) {
            if (src_lo == nullptr) CPB_TRY(launch_lo_plane(q.src, tl_lo_scratch, (long long)q.batch * q.src_img, s));
            return launch_tc_tapgemm(q, s);
        }
    }
    return launch_tapgemm(p, s);
}

static int32_t run_wgrad(const char* label, const float* big, int Wb, int pitch, long long big_img, int k,
                         const float* small, int B, int Ho, int Wo, int J, int c_pad, int c_real, float* partial,
                         float* out, cudaStream_t s) {
    ProfScope prof(label, s);
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = big; w.small = small; w.partial = partial;
    w.batch = B; w.Wb = Wb; w.big_pitch = pitch; w.big_img = big_img; w.Ho = Ho; w.Wo = Wo; w.sstride = 2;
    w.ntaps = k; w.run = k * pitch;
    for (int kh = 0; kh < k; ++kh) w.tap_off[kh] = (long long)kh * Wb * pitch;
    w.I = k * k * pitch; w.J = J;
    const long long M = (long long)B * Ho * Wo;
    if (g_math_mode == 1 && tc_wgrad_supported(w.I, w.J, w.run)) {
        w.splits = tc_wgrad_pick_splits(w.I, w.J, M);
        w.m_per_split = align_up((M + w.splits - 1) / w.splits, 32);
        CPB_TRY(launch_tc_wgrad(w, s));
    } else {
        w.splits = wgrad_pick_splits(w.I, w.J, M);
        w.m_per_split = align_up((M + w.splits - 1) / w.splits, 16);
        CPB_TRY(launch_wgrad(w, s));
    }
    return launch_reduce_partials(partial, w.splits, w.I, w.J, c_pad, c_real, out, s);
}

static int32_t run_dense_wgrad(const char* label, const float* x, int K, const float* g, int B, int J, float* partial,
                               float* out, cudaStream_t s) {
    ProfScope prof(label, s);
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = x; w.small = g; w.partial = partial;
    w.batch = B; w.Wb = 1; w.big_pitch = K; w.big_img = K; w.Ho = w.Wo = 1; w.sstride = 1;
    w.ntaps = 1; w.run = K; w.tap_off[0] = 0; w.I = K; w.J = J;
    w.splits = wgrad_pick_splits(w.I, w.J, B);
    w.m_per_split = align_up(((long long)B + w.splits - 1) / w.splits, 16);
    CPB_TRY(launch_wgrad(w, s));
    return launch_reduce_partials(partial, w.splits, w.I, w.J, K, K, out, s);
}

// ---------------------------------------------------------------------------------------------
// passes
// ---------------------------------------------------------------------------------------------
static int32_t check_cfg(const cpb_vae_config* cfg) {
    CPB_REQUIRE(cfg != nullptr, "cfg is NULL");
    CPB_REQUIRE(cfg->batch >= 1 && cfg->batch <= (1 << 20), "batch=%d out of range", cfg->batch);
    CPB_REQUIRE(cfg->target_channels == 1 || cfg->target_channels == 3, "target_channels must be 1 or 3, got %d", cfg->target_channels);
    CPB_REQUIRE(cfg->z_dim >= 64 && cfg->z_dim % 64 == 0 && cfg->z_dim <= 1024, "z_dim=%d must be a multiple of 64 in [64,1024]", cfg->z_dim);
    CPB_REQUIRE(cfg->loss_type >= 0 && cfg->loss_type <= 2, "unknown loss_type %d", cfg->loss_type);
    CPB_REQUIRE(cfg->source_dtype == CPB_FRAME_F32 || cfg->source_dtype == CPB_FRAME_U8, "bad source_dtype");
    CPB_REQUIRE(cfg->target_dtype == CPB_FRAME_F32 || cfg->target_dtype == CPB_FRAME_U8, "bad target_dtype");
    return CPB_OK;
}

static int32_t relayout_weights(const VaePlan& pl, const VaeLayout& L, const float* params, bool decoder,
                                bool backward, cudaStream_t s) {
    using namespace geo;
    RelayoutTable t;
    memset(&t, 0, sizeof(t));
    auto add = [&](int64_t src, int64_t dst, int taps, int rows, int cols, int mode, int rows_pad) {
        RelayoutJob& j = t.jobs[t.njobs++];
        j.src_off = src; j.dst_off = dst; j.taps = taps; j.rows = rows; j.cols = cols; j.mode = mode;
        j.rows_pad = rows_pad;
        j.count = mode == 0 ? (long long)taps * rows * cols : (long long)taps * rows_pad * cols;
        t.total += j.count;
    };
    if (decoder) {
        add(L.off[T_DECONV1_K], pl.rl.deconv1T, 16, C3, C4, 0, 0);
        add(L.off[T_DECONV2_K], pl.rl.deconv2T, 16, C2, C3, 0, 0);
        add(L.off[T_DECONV3_K], pl.rl.deconv3T, 25, C1, C2, 0, 0);
    }
    if (backward) {
        add(L.off[T_CONV2_K], pl.rl.conv2T, 16, C1, C2, 0, 0);
        add(L.off[T_CONV3_K], pl.rl.conv3T, 16, C2, C3, 0, 0);
        add(L.off[T_CONV4_K], pl.rl.conv4T, 16, C3, C4, 0, 0);
    }
    if (backward) {
        add(L.off[T_DENSE1_K], pl.rl.dense1T, 1, pl.z, FEAT, 0, 0);
        add(L.off[T_MEAN_K], pl.rl.headsT, 2, FEAT, pl.z, 0, 0);   // mean and logvar kernels are adjacent
    }
    ProfScope prof("relayout_weights", s);
    CPB_TRY(launch_relayout(params, pl.relayout, t, s));
    if (g_math_mode != 1) return CPB_OK;
    TcWeightTable w;
    memset(&w, 0, sizeof(w));
    auto addw = [&](int tensor, int slot, int k, int cb, int cs, bool gather, bool scatter) {
        const long long n = (long long)k * k * cb * cs;
        if (gather) {
            TcWeightJob& j = w.jobs[w.njobs++];
            j.src_off = L.off[tensor]; j.dst_hi = pl.rl.tc[slot].f_hi; j.dst_lo = pl.rl.tc[slot].f_lo;
            j.mode = 1; j.k = k; j.cb = cb; j.cs = cs; j.N = cs; j.C = k * cb; j.count = n; w.total += n;
        }
        if (scatter) {
            TcWeightJob& j = w.jobs[w.njobs++];
            j.src_off = L.off[tensor]; j.dst_hi = pl.rl.tc[slot].t_hi; j.dst_lo = pl.rl.tc[slot].t_lo;
            const int win = (k + 1) / 2;
            j.mode = 2; j.k = k; j.cb = cb; j.cs = cs; j.N = 4 * cb; j.C = cs; j.count = (long long)win * win * 4 * cb * cs; w.total += j.count;
        }
    };
    // conv layers run gather-form forward / scatter-form dgrad; deconv layers the other way round
    addw(T_CONV2_K, TC_CONV2, 4, C1, C2, true, backward);
    addw(T_CONV3_K, TC_CONV3, 4, C2, C3, true, backward);
    addw(T_CONV4_K, TC_CONV4, 4, C3, C4, true, backward);
    if (decoder) {
        addw(T_DECONV1_K, TC_DECONV1, 4, C3, C4, backward, true);
        addw(T_DECONV2_K, TC_DECONV2, 4, C2, C3, backward, true);
        addw(T_DECONV3_K, TC_DECONV3, 5, C1, C2, backward, true);
    }
    return launch_tc_weights(params, pl.relayout, w, s);
}

static int32_t run_encoder(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                           const void* source, int32_t* flags, cudaStream_t s) {
    tl_lo_scratch = pl.lo;
    using namespace geo;
    const int B = pl.B;
    const float sscale = cfg->source_dtype == CPB_FRAME_U8 ? 1.f / 255.f : 1.f;
    { ProfScope prof("prep_frames", s);
      CPB_TRY(launch_prep_frames(source, cfg->source_dtype, sscale, 3, (long long)B * NPIX, pl.xp, flags, 1, s)); }
    { ProfScope prof("conv1.fwd", s);
      CPB_TRY(launch_edge_gather(pl.xp, 3, params + L.off[T_CONV1_K], params + L.off[T_CONV1_B], nullptr, pl.a1,
                                 g_math_mode == 1 ? pl.a1_lo : nullptr, B, s)); }
    TapGemmParams p;
    p = gather_problem(pl.a1, B, H1, W1, C1, 4, params + L.off[T_CONV2_K], C2, params + L.off[T_CONV2_B], nullptr, pl.a2, 1,
                       pl.relayout + pl.rl.tc[TC_CONV2].f_hi, pl.relayout + pl.rl.tc[TC_CONV2].f_lo);
    CPB_TRY(tg("conv2.fwd", p, s, 0, pl.a1_lo, pl.a2_lo));
    p = gather_problem(pl.a2, B, H2, W2, C2, 4, params + L.off[T_CONV3_K], C3, params + L.off[T_CONV3_B], nullptr, pl.a3, 1,
                       pl.relayout + pl.rl.tc[TC_CONV3].f_hi, pl.relayout + pl.rl.tc[TC_CONV3].f_lo);
    CPB_TRY(tg("conv3.fwd", p, s, 0, pl.a2_lo, pl.a3_lo));
    p = gather_problem(pl.a3, B, H3, W3, C3, 4, params + L.off[T_CONV4_K], C4, params + L.off[T_CONV4_B], nullptr, pl.a4, 1,
                       pl.relayout + pl.rl.tc[TC_CONV4].f_hi, pl.relayout + pl.rl.tc[TC_CONV4].f_lo);
    CPB_TRY(tg("conv4.fwd", p, s, 0, pl.a3_lo, nullptr));
    // both heads as one y-batched dense problem: heads[0] = mean, heads[1] = logstd_sq
    p = dense_problem(pl.a4, B, FEAT, params + L.off[T_MEAN_K], pl.z, params + L.off[T_MEAN_B], nullptr, pl.heads, 0);
    p.ybatch = 2;
    p.w_ystride = L.off[T_LOGVAR_K] - L.off[T_MEAN_K];
    p.bias_ystride = L.off[T_LOGVAR_B] - L.off[T_MEAN_B];
    p.dst_ystride = (long long)B * pl.z;
    if (pl.z % 64 == 0) {
        p.ksplit = tapgemm_pick_ksplit(B, pl.z, 2, FEAT);
        p.kpartial = pl.ksplit; p.kpartial_stride = 2LL * B * pl.z;
    }
    return tg("heads.fwd", p, s);
}

// zbuf -> d1 -> b1 -> b2 -> b3 -> (logits_p and/or sigmoid)
static int32_t run_decoder(const VaePlan& pl, const VaeLayout& L, const float* params, const float* zsrc,
                           float* logits_p, float* sigm, cudaStream_t s) {
    tl_lo_scratch = pl.lo;
    using namespace geo;
    const int B = pl.B;
    TapGemmParams p = dense_problem(zsrc, B, pl.z, params + L.off[T_DENSE1_K], FEAT, params + L.off[T_DENSE1_B],
                                    nullptr, pl.d1, 0);
    CPB_TRY(tg("dense1.fwd", p, s));
    p = scatter_problem(pl.d1, B, H4, W4, C4, 4, pl.relayout + pl.rl.deconv1T, C3, params + L.off[T_DECONV1_B],
                        nullptr, pl.b1, H3, W3, 1, pl.relayout + pl.rl.tc[TC_DECONV1].t_hi, pl.relayout + pl.rl.tc[TC_DECONV1].t_lo);
    CPB_TRY(tg("deconv1.fwd", p, s, 4, nullptr, pl.b1_lo));
    p = scatter_problem(pl.b1, B, H3, W3, C3, 4, pl.relayout + pl.rl.deconv2T, C2, params + L.off[T_DECONV2_B],
                        nullptr, pl.b2, H2, W2, 1, pl.relayout + pl.rl.tc[TC_DECONV2].t_hi, pl.relayout + pl.rl.tc[TC_DECONV2].t_lo);
    CPB_TRY(tg("deconv2.fwd", p, s, 4, pl.b1_lo, pl.b2_lo));
    p = scatter_problem(pl.b2, B, H2, W2, C2, 5, pl.relayout + pl.rl.deconv3T, C1, params + L.off[T_DECONV3_B],
                        nullptr, pl.b3, H1, W1, 1, pl.relayout + pl.rl.tc[TC_DECONV3].t_hi, pl.relayout + pl.rl.tc[TC_DECONV3].t_lo);
    CPB_TRY(tg("deconv3.fwd", p, s, 5, pl.b2_lo, nullptr));
    ProfScope prof("deconv4.fwd", s);
    return launch_deconv4_fwd(pl.b3, params + L.off[T_DECONV4_K], params + L.off[T_DECONV4_B], B, pl.ct, logits_p,
                              sigm, s);
}

static int32_t run_forward_loss(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                                const void* source, const void* target, const float* eps, bool want_dlogits,
                                float* sigm, int32_t* flags, cudaStream_t s) {
    using namespace geo;
    const int B = pl.B;
    CPB_TRY(run_encoder(pl, L, cfg, params, source, flags, s));
    CPB_TRY(launch_reparam(pl.heads, eps, B, pl.z, cfg->kl_tolerance, pl.zbuf, pl.kl_rows, pl.kl_active, s));
    CPB_TRY(run_decoder(pl, L, params, pl.zbuf, pl.logits_p, sigm, s));
    const float* yp = pl.yp;
    if (target == source && cfg->target_channels == 3 && cfg->target_dtype == cfg->source_dtype &&
        (cfg->target_dtype == CPB_FRAME_F32 || cfg->target_u8_scale == 1.f / 255.f)) {
        yp = pl.xp;   // rgb target == source (vae/train_vae.py:75): already prepared and range-checked
    } else {
        const float tscale = cfg->target_dtype == CPB_FRAME_U8 ? cfg->target_u8_scale : 1.f;
        CPB_TRY(launch_prep_frames(target, cfg->target_dtype, tscale, cfg->target_channels, (long long)B * NPIX,
                                   pl.yp, flags, 2, s));
    }
    const float gscale = cfg->loss_scale / (float)B;
    { ProfScope prof("recon_loss", s);
      CPB_TRY(launch_recon_loss(pl.logits_p, yp, B, pl.ct, cfg->loss_type, gscale, pl.frame_loss,
                                want_dlogits ? pl.logits_p : nullptr, s, want_dlogits ? pl.frame_dsum : nullptr)); }
    return CPB_OK;
}

static int32_t run_backward(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                            const float* eps, float* grads, cudaStream_t s) {
    tl_lo_scratch = pl.lo;
    using namespace geo;
    const int B = pl.B;
    const int z = pl.z;
    float* dlog = pl.logits_p;   // overwritten in place by the loss kernel
    float* cs = pl.colsum;
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    // ---- deconv4 (padded to 4 channels on the big side)
    { ProfScope prof("deconv4.wgrad", s);
      CPB_TRY(launch_edge_wgrad(dlog, pl.ct, pl.b3, B, pl.partial, s));
      CPB_TRY(launch_reduce_partials(pl.partial, edge_wgrad_ctas(B), 16 * pl.ct, C1, 16 * pl.ct, 16 * pl.ct,
                                     grads + L.off[T_DECONV4_K], s)); }
    // the bias gradients of the two outermost layers come out of the kernels that write their pre-activation gradients
    // (recon_loss: per-frame channel sums; edge_gather: per-CTA column sums) instead of separate passes over 0.8 + 1.6 GB
    CPB_TRY(launch_colsum(pl.frame_dsum, B, 4, pl.ct, grads + L.off[T_DECONV4_B], cs, s));
    { ProfScope prof("deconv4.dgrad", s);
      CPB_TRY(launch_edge_gather(dlog, pl.ct, params + L.off[T_DECONV4_K], nullptr, pl.b3, pl.gA,
                                 g_math_mode == 1 ? pl.gA_lo : nullptr, B, s, pl.cs_edge)); }   // gA = g(b3 pre-activation)
    TapGemmParams p;
    // ---- deconv3
    CPB_TRY(run_wgrad("deconv3.wgrad", pl.gA, W1, C1, (long long)H1 * W1 * C1, 5, pl.b2, B, H2, W2, C2, 5 * 5 * C1, 5 * 5 * C1,
                      pl.partial, grads + L.off[T_DECONV3_K], s));
    CPB_TRY(launch_colsum(pl.cs_edge, edge_gather_blocks(B), C1, C1, grads + L.off[T_DECONV3_B], cs, s));
    p = gather_problem(pl.gA, B, H1, W1, C1, 5, params + L.off[T_DECONV3_K], C2, nullptr, pl.b2, pl.gB, 0,
                       pl.relayout + pl.rl.tc[TC_DECONV3].f_hi, pl.relayout + pl.rl.tc[TC_DECONV3].f_lo);
    CPB_TRY(tg("deconv3.dgrad", p, s, 0, pl.gA_lo, pl.gB_lo));   // gB = g(b2)
    // ---- deconv2
    CPB_TRY(run_wgrad("deconv2.wgrad", pl.gB, W2, C2, (long long)H2 * W2 * C2, 4, pl.b1, B, H3, W3, C3, 16 * C2, 16 * C2, pl.partial,
                      grads + L.off[T_DECONV2_K], s));
    CPB_TRY(launch_colsum(pl.gB, (long long)B * H2 * W2, C2, C2, grads + L.off[T_DECONV2_B], cs, s));
    p = gather_problem(pl.gB, B, H2, W2, C2, 4, params + L.off[T_DECONV2_K], C3, nullptr, pl.b1, pl.gA, 0,
                       pl.relayout + pl.rl.tc[TC_DECONV2].f_hi, pl.relayout + pl.rl.tc[TC_DECONV2].f_lo);
    CPB_TRY(tg("deconv2.dgrad", p, s, 0, pl.gB_lo, pl.gA_lo));   // gA = g(b1)
    // ---- deconv1
    CPB_TRY(run_wgrad("deconv1.wgrad", pl.gA, W3, C3, (long long)H3 * W3 * C3, 4, pl.d1, B, H4, W4, C4, 16 * C3, 16 * C3, pl.partial,
                      grads + L.off[T_DECONV1_K], s));
    CPB_TRY(launch_colsum(pl.gA, (long long)B * H3 * W3, C3, C3, grads + L.off[T_DECONV1_B], cs, s));
    p = gather_problem(pl.gA, B, H3, W3, C3, 4, params + L.off[T_DECONV1_K], C4, nullptr, nullptr, pl.gB, 0,
                       pl.relayout + pl.rl.tc[TC_DECONV1].f_hi, pl.relayout + pl.rl.tc[TC_DECONV1].f_lo);
    CPB_TRY(tg("deconv1.dgrad", p, s, 0, pl.gA_lo, nullptr));                                   // gB = g(d1) [B, 6144]
    // ---- dense1
    CPB_TRY(run_dense_wgrad("dense1.wgrad", pl.zbuf, z, pl.gB, B, FEAT, pl.partial, grads + L.off[T_DENSE1_K], s));
    CPB_TRY(launch_colsum(pl.gB, B, FEAT, FEAT, grads + L.off[T_DENSE1_B], cs, s));
    p = dense_problem(pl.gB, B, FEAT, pl.relayout + pl.rl.dense1T, z, nullptr, nullptr, pl.gz, 0);
    if (z % 64 == 0) {
        p.ksplit = tapgemm_pick_ksplit(B, z, 1, FEAT);
        p.kpartial = pl.ksplit; p.kpartial_stride = (long long)B * z;
    }
    CPB_TRY(tg("dense1.dgrad", p, s));
    // ---- sampling + KL
    CPB_TRY(launch_reparam_bwd(pl.heads, eps, pl.gz, pl.kl_active, B, z, cfg->beta * cfg->loss_scale / (float)B,
                               pl.gheads, s));
    // ---- heads
    CPB_TRY(run_dense_wgrad("heads.wgrad", pl.a4, FEAT, pl.gheads, B, z, pl.partial, grads + L.off[T_MEAN_K], s));
    CPB_TRY(run_dense_wgrad("heads.wgrad", pl.a4, FEAT, pl.gheads + (long long)B * z, B, z, pl.partial, grads + L.off[T_LOGVAR_K], s));
    CPB_TRY(launch_colsum(pl.gheads, B, z, z, grads + L.off[T_MEAN_B], cs, s));
    CPB_TRY(launch_colsum(pl.gheads + (long long)B * z, B, z, z, grads + L.off[T_LOGVAR_B], cs, s));
    p = dense_problem(pl.gheads, B, z, pl.relayout + pl.rl.headsT, FEAT, nullptr, pl.a4, pl.gA, 0);
    p.cls[0].ntaps = 2;                                              // g(a4) = gmean Wm^T + glogvar Wl^T
    p.cls[0].taps[1].dy = p.cls[0].taps[1].dx = 0;
    p.cls[0].taps[1].src_off = (long long)B * z;
    p.cls[0].taps[1].w_off = (long long)z * FEAT;
    CPB_TRY(tg("heads.dgrad", p, s));                                   // gA = g(a4 pre-activation)
    // ---- conv4
    CPB_TRY(run_wgrad("conv4.wgrad", pl.a3, W3, C3, (long long)H3 * W3 * C3, 4, pl.gA, B, H4, W4, C4, 16 * C3, 16 * C3, pl.partial,
                      grads + L.off[T_CONV4_K], s));
    CPB_TRY(launch_colsum(pl.gA, (long long)B * H4 * W4, C4, C4, grads + L.off[T_CONV4_B], cs, s));
    p = scatter_problem(pl.gA, B, H4, W4, C4, 4, pl.relayout + pl.rl.conv4T, C3, nullptr, pl.a3, pl.gB, H3, W3, 0,
                        pl.relayout + pl.rl.tc[TC_CONV4].t_hi, pl.relayout + pl.rl.tc[TC_CONV4].t_lo);
    CPB_TRY(tg("conv4.dgrad", p, s, 4, nullptr, pl.gB_lo));   // gB = g(a3)
    // ---- conv3
    CPB_TRY(run_wgrad("conv3.wgrad", pl.a2, W2, C2, (long long)H2 * W2 * C2, 4, pl.gB, B, H3, W3, C3, 16 * C2, 16 * C2, pl.partial,
                      grads + L.off[T_CONV3_K], s));
    CPB_TRY(launch_colsum(pl.gB, (long long)B * H3 * W3, C3, C3, grads + L.off[T_CONV3_B], cs, s));
    p = scatter_problem(pl.gB, B, H3, W3, C3, 4, pl.relayout + pl.rl.conv3T, C2, nullptr, pl.a2, pl.gA, H2, W2, 0,
                        pl.relayout + pl.rl.tc[TC_CONV3].t_hi, pl.relayout + pl.rl.tc[TC_CONV3].t_lo);
    CPB_TRY(tg("conv3.dgrad", p, s, 4, pl.gB_lo, pl.gA_lo));   // gA = g(a2)
    // ---- conv2
    CPB_TRY(run_wgrad("conv2.wgrad", pl.a1, W1, C1, (long long)H1 * W1 * C1, 4, pl.gA, B, H2, W2, C2, 16 * C1, 16 * C1, pl.partial,
                      grads + L.off[T_CONV2_K], s));
    CPB_TRY(launch_colsum(pl.gA, (long long)B * H2 * W2, C2, C2, grads + L.off[T_CONV2_B], cs, s));
    p = scatter_problem(pl.gA, B, H2, W2, C2, 4, pl.relayout + pl.rl.conv2T, C1, nullptr, pl.a1, pl.gB, H1, W1, 0,
                        pl.relayout + pl.rl.tc[TC_CONV2].t_hi, pl.relayout + pl.rl.tc[TC_CONV2].t_lo);
    CPB_TRY(tg("conv2.dgrad", p, s, 4, pl.gA_lo, nullptr));   // gB = g(a1)
    // ---- conv1 (its input gradient is never used: the reference computes and discards it)
    { ProfScope prof("conv1.wgrad", s);
      CPB_TRY(launch_edge_wgrad(pl.xp, 3, pl.gB, B, pl.partial, s));
      CPB_TRY(launch_reduce_partials(pl.partial, edge_wgrad_ctas(B), 48, C1, 48, 48, grads + L.off[T_CONV1_K], s)); }
    CPB_TRY(launch_colsum(pl.gB, (long long)B * H1 * W1, C1, C1, grads + L.off[T_CONV1_B], cs, s));
    return CPB_OK;
}


// =============================================================================================
// MlpVAE (reference vae/models.py:271-299): flatten -> dense E1 relu -> dense E2 relu -> [mean | logstd_sq] -> sample ->
// dense D1 relu -> dense D2 relu -> dense 12800*Ct -> logits.  Same loss / sampling / Adam kernels as the ConvVAE; all
// seven layers run on the fp32 SIMT tap-GEMM (dense form) and the SIMT weight-gradient kernel.
// =============================================================================================
enum MlpTensor { M_E1_K, M_E1_B, M_E2_K, M_E2_B, M_MEAN_K, M_MEAN_B, M_LOGVAR_K, M_LOGVAR_B, M_D1_K, M_D1_B, M_D2_K, M_D2_B, M_D3_K, M_D3_B, M_COUNT };
static const char* kMlpNames[M_COUNT] = {
    "encoder/dense/kernel", "encoder/dense/bias", "encoder/dense_1/kernel", "encoder/dense_1/bias",
    "mean/kernel", "mean/bias", "logstd_sqare/kernel", "logstd_sqare/bias",
    "decoder/dense/kernel", "decoder/dense/bias", "decoder/dense_1/kernel", "decoder/dense_1/bias",
    "decoder/dense_2/kernel", "decoder/dense_2/bias"};

struct MlpLayout { int64_t off[M_COUNT], size[M_COUNT]; int32_t shape[M_COUNT][2]; int64_t total; };

static int32_t check_mlp_cfg(const cpb_mlpvae_config* c) {
    CPB_REQUIRE(c != nullptr, "mlp cfg is NULL");
    CPB_TRY(check_cfg(&c->base));
    for (int v : {c->enc1, c->enc2, c->dec1, c->dec2})
        CPB_REQUIRE(v >= 32 && v % 32 == 0 && v <= 8192, "MlpVAE hidden sizes must be multiples of 32 in [32, 8192], got %d", v);
    return CPB_OK;
}

static MlpLayout make_mlp_layout(const cpb_mlpvae_config* c) {
    const int IN = geo::NPIX * 3, OUT = geo::NPIX * c->base.target_channels, z = c->base.z_dim;
    const int shp[M_COUNT][2] = {{IN, c->enc1}, {c->enc1, 0}, {c->enc1, c->enc2}, {c->enc2, 0}, {c->enc2, z}, {z, 0}, {c->enc2, z}, {z, 0},
                                 {z, c->dec1}, {c->dec1, 0}, {c->dec1, c->dec2}, {c->dec2, 0}, {c->dec2, OUT}, {OUT, 0}};
    // the two head kernels (and biases) adjacent: both heads run as one y-batched dense problem
    static const int order[M_COUNT] = {M_E1_K, M_E1_B, M_E2_K, M_E2_B, M_MEAN_K, M_LOGVAR_K, M_MEAN_B, M_LOGVAR_B,
                                       M_D1_K, M_D1_B, M_D2_K, M_D2_B, M_D3_K, M_D3_B};
    MlpLayout L;
    for (int i = 0; i < M_COUNT; ++i) { L.shape[i][0] = shp[i][0]; L.shape[i][1] = shp[i][1]; L.size[i] = (int64_t)shp[i][0] * (shp[i][1] ? shp[i][1] : 1); }
    int64_t o = 0;
    for (int i = 0; i < M_COUNT; ++i) { L.off[order[i]] = o; o += align_up(L.size[order[i]], 64); }
    L.total = o;
    return L;
}

struct MlpPlan {
    int B, IN, OUT, z, e1, e2, d1, d2;
    float *x, *y, *h1, *h2, *heads, *zbuf, *kl_rows, *kl_active, *frame_loss, *g1, *g2, *logits;
    float *ga, *gb, *gz, *gheads, *partial, *colsum, *wT, *ksplit;
    int64_t tE2, tHeads, tD1, tD2, tD3;      // float offsets of the transposed kernels inside wT
    int64_t bytes;
    bool ok;
};

static MlpPlan make_mlp_plan(void* ws, int64_t ws_bytes, const cpb_mlpvae_config* c, int mode) {
    MlpPlan p;
    memset(&p, 0, sizeof(p));
    const int64_t b = c->base.batch;
    p.B = (int)b; p.IN = geo::NPIX * 3; p.OUT = geo::NPIX * c->base.target_channels; p.z = c->base.z_dim;
    p.e1 = c->enc1; p.e2 = c->enc2; p.d1 = c->dec1; p.d2 = c->dec2;
    Arena a(ws, ws_bytes);
    p.x = a.take<float>(b * p.IN);
    p.h1 = a.take<float>(b * p.e1);
    p.h2 = a.take<float>(b * p.e2);
    p.heads = a.take<float>(2 * b * p.z);
    p.ksplit = a.take<float>((int64_t)kMaxKSplit * 2 * b * p.z);
    if (mode >= CPB_WS_FORWARD) {
        p.y = a.take<float>(b * p.OUT);
        p.zbuf = a.take<float>(b * p.z);
        p.kl_rows = a.take<float>(b); p.kl_active = a.take<float>(b); p.frame_loss = a.take<float>(b);
        p.g1 = a.take<float>(b * p.d1);
        p.g2 = a.take<float>(b * p.d2);
        p.logits = a.take<float>(b * p.OUT);
    }
    if (mode >= CPB_WS_TRAIN) {
        const int64_t widest = std::max<int64_t>(std::max(p.e1, p.e2), std::max(p.d1, p.d2));
        p.ga = a.take<float>(b * widest);
        p.gb = a.take<float>(b * widest);
        p.gz = a.take<float>(b * p.z);
        p.gheads = a.take<float>(2 * b * p.z);
        int64_t o = 0;
        auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
        p.tE2 = take((int64_t)p.e1 * p.e2); p.tHeads = take(2LL * p.e2 * p.z); p.tD1 = take((int64_t)p.z * p.d1);
        p.tD2 = take((int64_t)p.d1 * p.d2); p.tD3 = take((int64_t)p.d2 * p.OUT);
        p.wT = a.take<float>(o);
        struct P { int I, J; };
        const P ps[] = {{p.IN, p.e1}, {p.e1, p.e2}, {p.e2, p.z}, {p.z, p.d1}, {p.d1, p.d2}, {p.d2, p.OUT}};
        int64_t best = 0;
        for (const P& q : ps) best = std::max<int64_t>(best, (int64_t)wgrad_pick_splits(q.I, q.J, b) * q.I * q.J);
        p.partial = a.take<float>(best);
        p.colsum = a.take<float>(colsum_scratch_floats(b, p.OUT) + colsum_scratch_floats(b, (int)widest));
    }
    p.bytes = a.off;
    p.ok = ws == nullptr || !a.overflow;
    return p;
}

static int32_t mlp_encoder(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_config* c, const float* params, const void* source,
                           int32_t* flags, cudaStream_t s) {
    const float sscale = c->base.source_dtype == CPB_FRAME_U8 ? 1.f / 255.f : 1.f;
    CPB_TRY(launch_prep_flat(source, c->base.source_dtype, sscale, (long long)pl.B * pl.IN, pl.x, flags, 1, s));
    TapGemmParams p = dense_problem(pl.x, pl.B, pl.IN, params + L.off[M_E1_K], pl.e1, params + L.off[M_E1_B], nullptr, pl.h1, 1);
    CPB_TRY(launch_tapgemm(p, s));
    p = dense_problem(pl.h1, pl.B, pl.e1, params + L.off[M_E2_K], pl.e2, params + L.off[M_E2_B], nullptr, pl.h2, 1);
    CPB_TRY(launch_tapgemm(p, s));
    p = dense_problem(pl.h2, pl.B, pl.e2, params + L.off[M_MEAN_K], pl.z, params + L.off[M_MEAN_B], nullptr, pl.heads, 0);
    p.ybatch = 2;
    p.w_ystride = L.off[M_LOGVAR_K] - L.off[M_MEAN_K];
    p.bias_ystride = L.off[M_LOGVAR_B] - L.off[M_MEAN_B];
    p.dst_ystride = (long long)pl.B * pl.z;
    return launch_tapgemm(p, s);
}

static int32_t mlp_decoder(const MlpPlan& pl, const MlpLayout& L, const float* params, const float* zsrc, float* logits, cudaStream_t s) {
    TapGemmParams p = dense_problem(zsrc, pl.B, pl.z, params + L.off[M_D1_K], pl.d1, params + L.off[M_D1_B], nullptr, pl.g1, 1);
    CPB_TRY(launch_tapgemm(p, s));
    p = dense_problem(pl.g1, pl.B, pl.d1, params + L.off[M_D2_K], pl.d2, params + L.off[M_D2_B], nullptr, pl.g2, 1);
    CPB_TRY(launch_tapgemm(p, s));
    p = dense_problem(pl.g2, pl.B, pl.d2, params + L.off[M_D3_K], pl.OUT, params + L.off[M_D3_B], nullptr, logits, 0);
    return launch_tapgemm(p, s);
}

static int32_t mlp_forward_loss(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_config* c, const float* params, const void* source,
                                const void* target, const float* eps, bool want_dlogits, int32_t* flags, cudaStream_t s) {
    CPB_TRY(mlp_encoder(pl, L, c, params, source, flags, s));
    CPB_TRY(launch_reparam(pl.heads, eps, pl.B, pl.z, c->base.kl_tolerance, pl.zbuf, pl.kl_rows, pl.kl_active, s));
    CPB_TRY(mlp_decoder(pl, L, params, pl.zbuf, pl.logits, s));
    const float* y = pl.y;
    if (target == source && c->base.target_channels == 3 && c->base.target_dtype == c->base.source_dtype &&
        (c->base.target_dtype == CPB_FRAME_F32 || c->base.target_u8_scale == 1.f / 255.f)) {
        y = pl.x;
    } else {
        const float tscale = c->base.target_dtype == CPB_FRAME_U8 ? c->base.target_u8_scale : 1.f;
        CPB_TRY(launch_prep_flat(target, c->base.target_dtype, tscale, (long long)pl.B * pl.OUT, pl.y, flags, 2, s));
    }
    return launch_recon_loss_flat(pl.logits, y, pl.B, pl.OUT, c->base.loss_type, c->base.loss_scale / (float)pl.B, pl.frame_loss,
                                  want_dlogits ? pl.logits : nullptr, s);
}

static int32_t mlp_backward(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_config* c, const float* params, const float* eps,
                            float* grads, cudaStream_t s) {
    const int B = pl.B, z = pl.z;
    float* dlog = pl.logits;
    float* cs = pl.colsum;
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    // transposed kernels for the data gradients ([in,out] -> [out,in]); the two head kernels are adjacent (2 "taps")
    RelayoutTable t;
    memset(&t, 0, sizeof(t));
    auto add = [&](int64_t src, int64_t dst, int taps, int rows, int cols) {
        RelayoutJob& j = t.jobs[t.njobs++];
        j.src_off = src; j.dst_off = dst; j.taps = taps; j.rows = rows; j.cols = cols; j.mode = 0; j.rows_pad = 0;
        j.count = (long long)taps * rows * cols; t.total += j.count;
    };
    add(L.off[M_E2_K], pl.tE2, 1, pl.e1, pl.e2);
    add(L.off[M_MEAN_K], pl.tHeads, 2, pl.e2, z);
    add(L.off[M_D1_K], pl.tD1, 1, z, pl.d1);
    add(L.off[M_D2_K], pl.tD2, 1, pl.d1, pl.d2);
    add(L.off[M_D3_K], pl.tD3, 1, pl.d2, pl.OUT);
    CPB_TRY(launch_relayout(params, pl.wT, t, s));
    TapGemmParams p;
    // ---- decoder
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.g2, pl.d2, dlog, B, pl.OUT, pl.partial, grads + L.off[M_D3_K], s));
    CPB_TRY(launch_colsum(dlog, B, pl.OUT, pl.OUT, grads + L.off[M_D3_B], cs, s));
    p = dense_problem(dlog, B, pl.OUT, pl.wT + pl.tD3, pl.d2, nullptr, pl.g2, pl.ga, 0);                       // ga = g(g2 pre-activation)
    CPB_TRY(launch_tapgemm(p, s));
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.g1, pl.d1, pl.ga, B, pl.d2, pl.partial, grads + L.off[M_D2_K], s));
    CPB_TRY(launch_colsum(pl.ga, B, pl.d2, pl.d2, grads + L.off[M_D2_B], cs, s));
    p = dense_problem(pl.ga, B, pl.d2, pl.wT + pl.tD2, pl.d1, nullptr, pl.g1, pl.gb, 0);                         // gb = g(g1 pre-activation)
    CPB_TRY(launch_tapgemm(p, s));
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.zbuf, z, pl.gb, B, pl.d1, pl.partial, grads + L.off[M_D1_K], s));
    CPB_TRY(launch_colsum(pl.gb, B, pl.d1, pl.d1, grads + L.off[M_D1_B], cs, s));
    p = dense_problem(pl.gb, B, pl.d1, pl.wT + pl.tD1, z, nullptr, nullptr, pl.gz, 0);
    CPB_TRY(launch_tapgemm(p, s));
    // ---- sampling + KL, heads
    CPB_TRY(launch_reparam_bwd(pl.heads, eps, pl.gz, pl.kl_active, B, z, c->base.beta * c->base.loss_scale / (float)B, pl.gheads, s));
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.h2, pl.e2, pl.gheads, B, z, pl.partial, grads + L.off[M_MEAN_K], s));
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.h2, pl.e2, pl.gheads + (long long)B * z, B, z, pl.partial, grads + L.off[M_LOGVAR_K], s));
    CPB_TRY(launch_colsum(pl.gheads, B, z, z, grads + L.off[M_MEAN_B], cs, s));
    CPB_TRY(launch_colsum(pl.gheads + (long long)B * z, B, z, z, grads + L.off[M_LOGVAR_B], cs, s));
    p = dense_problem(pl.gheads, B, z, pl.wT + pl.tHeads, pl.e2, nullptr, pl.h2, pl.ga, 0);
    p.cls[0].ntaps = 2;
    p.cls[0].taps[1].dy = p.cls[0].taps[1].dx = 0;
    p.cls[0].taps[1].src_off = (long long)B * z;
    p.cls[0].taps[1].w_off = (long long)z * pl.e2;
    CPB_TRY(launch_tapgemm(p, s));                                                                               // ga = g(h2 pre-activation)
    // ---- encoder
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.h1, pl.e1, pl.ga, B, pl.e2, pl.partial, grads + L.off[M_E2_K], s));
    CPB_TRY(launch_colsum(pl.ga, B, pl.e2, pl.e2, grads + L.off[M_E2_B], cs, s));
    p = dense_problem(pl.ga, B, pl.e2, pl.wT + pl.tE2, pl.e1, nullptr, pl.h1, pl.gb, 0);                         // gb = g(h1 pre-activation)
    CPB_TRY(launch_tapgemm(p, s));
    CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.x, pl.IN, pl.gb, B, pl.e1, pl.partial, grads + L.off[M_E1_K], s));
    return launch_colsum(pl.gb, B, pl.e1, pl.e1, grads + L.off[M_E1_B], cs, s);
}

}  // namespace cpb

// =============================================================================================
// C ABI
// =============================================================================================
using namespace cpb;

extern "C" {

const char* cpb_last_error(void) { return cpb::g_err; }
const char* cpb_build_info(void) { return "carla_ppo_b200 0.3 (sm_90a; wgmma 3xTF32 + fp32 SIMT tap-GEMM)"; }
int64_t cpb_launch_count(void) { return cpb::g_launches; }
void cpb_reset_launch_count(void) { cpb::g_launches = 0; }

/* debug: byte offsets of the named workspace buffers for (batch, ct, z, mode); returns the count written */
int32_t cpb_debug_vae_buffer_offsets(int32_t batch, int32_t ct, int32_t z, int32_t mode, int64_t* offsets, int32_t capacity) {
    char* base = (char*)4096;   // fake non-null base: only differences are used
    VaePlan pl = make_plan(base, (int64_t)1 << 60, batch, ct, z, mode);
    const float* ptrs[] = {pl.xp, pl.a1, pl.a2, pl.a3, pl.a4, pl.heads, pl.zbuf, pl.d1, pl.b1, pl.b2, pl.b3, pl.logits_p, pl.gA, pl.gB,
                           pl.frame_loss, pl.kl_rows};
    const int n = (int)(sizeof(ptrs) / sizeof(ptrs[0]));
    for (int i = 0; i < n && i < capacity; ++i) offsets[i] = ptrs[i] ? (int64_t)((const char*)ptrs[i] - base) : -1;
    return n;
}

/* debug: D[M,N] = A[M,K] * Bt[N,K]^T through the tensor-core tap-GEMM (dense, one tap).  scratch: 2*N*K + M*K floats. */
int32_t cpb_debug_tc_gemm(const float* a, const float* bt, float* d, int32_t m, int32_t n, int32_t k, float* scratch, void* stream) {
    CPB_TRY(ensure_init());
    cudaStream_t s = (cudaStream_t)stream;
    TcWeightTable w;
    memset(&w, 0, sizeof(w));
    w.njobs = 1; w.total = (long long)n * k;
    w.jobs[0].src_off = 0; w.jobs[0].dst_hi = 0; w.jobs[0].dst_lo = (long long)n * k; w.jobs[0].mode = 0; w.jobs[0].N = n; w.jobs[0].C = k; w.jobs[0].count = w.total;
    TapGemmParams p = dense_problem(a, m, k, nullptr, n, nullptr, nullptr, d, 0);
    p.wk_hi = scratch; p.wk_lo = scratch + (long long)n * k;
    p.debug = tc_debug_flags();
    CPB_TRY(launch_tc_weights(bt, scratch, w, s));
    float* lo = scratch + 2LL * n * k;
    p.src_lo = lo;
    CPB_TRY(launch_lo_plane(a, lo, (long long)m * k, s));
    return launch_tc_tapgemm(p, s);
}

/* debug: out[I,J] = big[M,I]^T small[M,J] through the tensor-core wgrad kernel (1x1 "image", one tap). */
int32_t cpb_debug_tc_wgrad(const float* big, const float* small, float* out, int32_t m, int32_t i, int32_t j,
                           int32_t variant, float* partial, void* stream) {
    CPB_TRY(ensure_init());
    cudaStream_t s = (cudaStream_t)stream;
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = big; w.small = small; w.partial = partial;
    w.batch = m; w.Wb = 1; w.big_pitch = i; w.big_img = i; w.Ho = w.Wo = 1; w.sstride = 1;
    w.ntaps = 1; w.run = i; w.tap_off[0] = 0; w.I = i; w.J = j; w.tc_variant = variant;
    w.splits = 2;
    w.m_per_split = align_up(((long long)m + 1) / 2, 32);
    CPB_TRY(launch_tc_wgrad(w, s));
    return launch_reduce_partials(partial, w.splits, i, j, i, i, out, s);
}

int32_t cpb_set_math_mode(int32_t mode) {
    CPB_REQUIRE(mode == 0 || mode == 1, "math mode must be 0 (fp32 SIMT) or 1 (3xTF32 wgmma)");
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

int32_t cpb_vae_num_tensors(void) { return T_COUNT; }
const char* cpb_vae_tensor_name(int32_t i) { return (i >= 0 && i < T_COUNT) ? kVaeNames[i] : nullptr; }

int32_t cpb_vae_layout(int32_t ct, int32_t z, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_REQUIRE(ct == 1 || ct == 3, "target_channels must be 1 or 3, got %d", ct);
    CPB_REQUIRE(z >= 64 && z % 64 == 0 && z <= 1024, "z_dim=%d must be a multiple of 64 in [64,1024]", z);
    VaeLayout L = make_layout(ct, z);
    for (int i = 0; i < T_COUNT; ++i) {
        if (offsets) offsets[i] = L.off[i];
        if (sizes) sizes[i] = L.size[i];
        if (shapes) for (int d = 0; d < 4; ++d) shapes[i * 4 + d] = L.shape[i][d];
    }
    if (total) *total = L.total;
    return CPB_OK;
}

int64_t cpb_vae_workspace_bytes(int32_t batch, int32_t ct, int32_t z, int32_t mode) {
    if (batch < 1 || (ct != 1 && ct != 3) || z < 64 || z % 64 != 0 || mode < 0 || mode > 2) {
        cpb::set_error("cpb_vae_workspace_bytes: bad arguments");
        return CPB_ERR_INVALID_ARGUMENT;
    }
    return make_plan(nullptr, 0, batch, ct, z, mode).bytes;
}

#define CPB_PLAN(mode)                                                                              \
    CPB_TRY(check_cfg(cfg));                                                                        \
    CPB_TRY(ensure_init());                                                                         \
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");                                         \
    VaePlan pl = make_plan(workspace, workspace_bytes, cfg->batch, cfg->target_channels, cfg->z_dim, mode); \
    if (!pl.ok) {                                                                                   \
        cpb::set_error("workspace too small: need %lld bytes, got %lld", (long long)pl.bytes,       \
                       (long long)workspace_bytes);                                                 \
        return CPB_ERR_WORKSPACE_TOO_SMALL;                                                         \
    }                                                                                               \
    VaeLayout L = make_layout(cfg->target_channels, cfg->z_dim);                                    \
    cudaStream_t s = (cudaStream_t)stream;

int32_t cpb_vae_encode(const cpb_vae_config* cfg, const float* params, const void* source, float* mean,
                       float* logvar, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PLAN(CPB_WS_ENCODE);
    CPB_REQUIRE(params && source && mean, "encode: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, false, false, s));
    CPB_TRY(run_encoder(pl, L, cfg, params, source, flags, s));
    const size_t n = (size_t)pl.B * pl.z * sizeof(float);
    CPB_CUDA(cudaMemcpyAsync(mean, pl.heads, n, cudaMemcpyDeviceToDevice, s));
    if (logvar) CPB_CUDA(cudaMemcpyAsync(logvar, pl.heads + (long long)pl.B * pl.z, n, cudaMemcpyDeviceToDevice, s));
    return CPB_OK;
}

int32_t cpb_vae_decode(const cpb_vae_config* cfg, const float* params, const float* z, float* reconstruction,
                       void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && z && reconstruction, "decode: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, false, s));
    return run_decoder(pl, L, params, z, nullptr, reconstruction, s);
}

int32_t cpb_vae_forward(const cpb_vae_config* cfg, const float* params, const void* source, const void* target,
                        const float* eps, float* losses, float* mean, float* logvar, float* z,
                        float* reconstruction, int32_t* flags, void* workspace, int64_t workspace_bytes,
                        void* stream) {
    CPB_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && source && target && losses, "forward: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, false, s));
    CPB_TRY(run_forward_loss(pl, L, cfg, params, source, target, eps, false, reconstruction, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, cfg->loss_scale, losses, s));
    const size_t n = (size_t)pl.B * pl.z * sizeof(float);
    if (mean) CPB_CUDA(cudaMemcpyAsync(mean, pl.heads, n, cudaMemcpyDeviceToDevice, s));
    if (logvar) CPB_CUDA(cudaMemcpyAsync(logvar, pl.heads + (long long)pl.B * pl.z, n, cudaMemcpyDeviceToDevice, s));
    if (z) CPB_CUDA(cudaMemcpyAsync(z, pl.zbuf, n, cudaMemcpyDeviceToDevice, s));
    return CPB_OK;
}

int32_t cpb_vae_loss_grad(const cpb_vae_config* cfg, const float* params, const void* source, const void* target,
                          const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_PLAN(CPB_WS_TRAIN);
    CPB_REQUIRE(params && source && target && grads && losses, "loss_grad: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, true, s));
    CPB_TRY(run_forward_loss(pl, L, cfg, params, source, target, eps, true, nullptr, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, cfg->loss_scale, losses, s));
    return run_backward(pl, L, cfg, params, eps, grads, s);
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

int32_t cpb_vae_train_step(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m, float* adam_v,
                           float* adam_powers, float lr, const void* source, const void* target, const float* eps,
                           float* losses, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_TRY(cpb_vae_loss_grad(cfg, params, source, target, eps, grads, losses, flags, workspace, workspace_bytes, stream));
    VaeLayout L = make_layout(cfg->target_channels, cfg->z_dim);
    // verify_range (vae/models.py:24-30, 89-90) is a tf.Assert the train op depends on: an out-of-range batch aborts the
    // reference's sess.run BEFORE ApplyAdam.  Same here: the update is skipped on the device when a flag bit is set.
    return cpb_adam_apply_guarded(params, grads, adam_m, adam_v, L.total, adam_powers, lr, nullptr, 0.9f, 0.999f, 1e-8f, flags, stream);
}

// state[b, 0:z] = latent[b, 0:z]; state[b, z:z+M] = measurements[b, 0:M]   (vae_common.py:59-61: np.append(encoded_state, measurements))
__global__ void assemble_state_kernel(const float* __restrict__ latent, const float* __restrict__ meas, int batch, int z, int m,
                                      float* __restrict__ state) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int w = z + m;
    if (idx >= batch * w) return;
    const int b = idx / w, c = idx - b * w;
    state[idx] = c < z ? latent[b * z + c] : meas[b * m + (c - z)];
}

int32_t cpb_encode_predict(const cpb_vae_config* vae_cfg, const float* vae_params, const void* frames, const float* measurements,
                           int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                           float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                           int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    CPB_REQUIRE(vae_cfg && ppo_cfg && frames && latent_tmp && state && action && value, "encode_predict: NULL pointer");
    CPB_REQUIRE(num_measurements >= 0 && (num_measurements == 0 || measurements != nullptr), "encode_predict: bad measurements");
    CPB_REQUIRE(ppo_cfg->state_dim == vae_cfg->z_dim + num_measurements, "encode_predict: state_dim %d != z_dim %d + %d measurements",
                ppo_cfg->state_dim, vae_cfg->z_dim, num_measurements);
    const int B = vae_cfg->batch;
    CPB_TRY(cpb_vae_encode(vae_cfg, vae_params, frames, latent_tmp, nullptr, flags, vae_workspace, vae_workspace_bytes, stream));
    const int total = B * ppo_cfg->state_dim;
    assemble_state_kernel<<<cdiv(total, 128), 128, 0, (cudaStream_t)stream>>>(latent_tmp, measurements, B, vae_cfg->z_dim, num_measurements, state);
    CPB_LAUNCHED();
    return cpb_ppo_forward(ppo_cfg, ppo_params, state, B, noise, action, value, ppo_workspace, ppo_workspace_bytes, stream);
}

static int64_t frame_bytes(int dtype, int channels) {
    return (int64_t)geo::NPIX * channels * (dtype == CPB_FRAME_U8 ? 1 : 4);
}

int64_t cpb_vae_staging_bytes(const cpb_vae_config* cfg) {
    if (check_cfg(cfg) != CPB_OK) return CPB_ERR_INVALID_ARGUMENT;
    const int64_t b = cfg->batch;
    return align_up(b * frame_bytes(cfg->source_dtype, 3), 256) +
           align_up(b * frame_bytes(cfg->target_dtype, cfg->target_channels), 256) +
           align_up(b * cfg->z_dim * 4, 256) + 256;
}

int32_t cpb_vae_train_step_host(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, float lr, const void* source_host,
                                const void* target_host, const float* eps_host, float* losses_host,
                                int32_t* flags_host, void* staging, int64_t staging_bytes, void* workspace,
                                int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_cfg(cfg));
    CPB_REQUIRE(source_host && target_host && eps_host && losses_host && staging, "train_step_host: NULL pointer");
    CPB_REQUIRE(staging_bytes >= cpb_vae_staging_bytes(cfg), "staging buffer too small");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t b = cfg->batch;
    Arena a(staging, staging_bytes);
    const int64_t sb = b * frame_bytes(cfg->source_dtype, 3);
    const int64_t tb = b * frame_bytes(cfg->target_dtype, cfg->target_channels);
    char* d_src = a.take<char>(sb);
    char* d_tgt = a.take<char>(tb);
    float* d_eps = a.take<float>(b * cfg->z_dim);
    float* d_out = a.take<float>(4);   // losses[2], flags
    CPB_CUDA(cudaMemcpyAsync(d_src, source_host, sb, cudaMemcpyHostToDevice, s));
    const void* tgt = d_src;
    if (target_host != source_host) {
        CPB_CUDA(cudaMemcpyAsync(d_tgt, target_host, tb, cudaMemcpyHostToDevice, s));
        tgt = d_tgt;
    }
    CPB_CUDA(cudaMemcpyAsync(d_eps, eps_host, b * cfg->z_dim * 4, cudaMemcpyHostToDevice, s));
    CPB_CUDA(cudaMemsetAsync(d_out, 0, 16, s));
    CPB_TRY(cpb_vae_train_step(cfg, params, grads, adam_m, adam_v, adam_powers, lr, d_src, tgt, d_eps, d_out,
                               (int32_t*)(d_out + 2), workspace, workspace_bytes, stream));
    float host_out[4];
    CPB_CUDA(cudaMemcpyAsync(host_out, d_out, 16, cudaMemcpyDeviceToHost, s));
    CPB_CUDA(cudaStreamSynchronize(s));
    losses_host[0] = host_out[0];
    losses_host[1] = host_out[1];
    if (flags_host) memcpy(flags_host, &host_out[2], 4);
    return CPB_OK;
}

/* ---------------------------------------------------------------------------------------------------- MlpVAE */
int32_t cpb_mlpvae_num_tensors(void) { return M_COUNT; }
const char* cpb_mlpvae_tensor_name(int32_t i) { return (i >= 0 && i < M_COUNT) ? kMlpNames[i] : nullptr; }

int32_t cpb_mlpvae_layout(const cpb_mlpvae_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_TRY(check_mlp_cfg(cfg));
    MlpLayout L = make_mlp_layout(cfg);
    for (int i = 0; i < M_COUNT; ++i) {
        if (offsets) offsets[i] = L.off[i];
        if (sizes) sizes[i] = L.size[i];
        if (shapes) { shapes[i * 4] = L.shape[i][0]; shapes[i * 4 + 1] = L.shape[i][1]; shapes[i * 4 + 2] = 0; shapes[i * 4 + 3] = 0; }
    }
    if (total) *total = L.total;
    return CPB_OK;
}

int64_t cpb_mlpvae_workspace_bytes(const cpb_mlpvae_config* cfg, int32_t mode) {
    if (check_mlp_cfg(cfg) != CPB_OK || mode < 0 || mode > 2) return CPB_ERR_INVALID_ARGUMENT;
    return make_mlp_plan(nullptr, 0, cfg, mode).bytes;
}

#define CPB_MLP_PLAN(mode)                                                                           \
    CPB_TRY(check_mlp_cfg(cfg));                                                                     \
    CPB_TRY(ensure_init());                                                                          \
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");                                          \
    MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, cfg, mode);                               \
    if (!pl.ok) {                                                                                    \
        cpb::set_error("workspace too small: need %lld bytes, got %lld", (long long)pl.bytes, (long long)workspace_bytes); \
        return CPB_ERR_WORKSPACE_TOO_SMALL;                                                          \
    }                                                                                                \
    MlpLayout L = make_mlp_layout(cfg);                                                              \
    cudaStream_t s = (cudaStream_t)stream;

int32_t cpb_mlpvae_encode(const cpb_mlpvae_config* cfg, const float* params, const void* source, float* mean, float* logvar,
                          int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_ENCODE);
    CPB_REQUIRE(params && source && mean, "mlp encode: NULL pointer");
    CPB_TRY(mlp_encoder(pl, L, cfg, params, source, flags, s));
    const size_t n = (size_t)pl.B * pl.z * sizeof(float);
    CPB_CUDA(cudaMemcpyAsync(mean, pl.heads, n, cudaMemcpyDeviceToDevice, s));
    if (logvar) CPB_CUDA(cudaMemcpyAsync(logvar, pl.heads + (long long)pl.B * pl.z, n, cudaMemcpyDeviceToDevice, s));
    return CPB_OK;
}

int32_t cpb_mlpvae_decode(const cpb_mlpvae_config* cfg, const float* params, const float* z, float* reconstruction, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && z && reconstruction, "mlp decode: NULL pointer");
    CPB_TRY(mlp_decoder(pl, L, params, z, pl.logits, s));
    return launch_sigmoid(pl.logits, reconstruction, (long long)pl.B * pl.OUT, s);
}

int32_t cpb_mlpvae_forward(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target, const float* eps,
                           float* losses, float* mean, float* logvar, float* z, float* reconstruction, int32_t* flags,
                           void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && source && target && losses, "mlp forward: NULL pointer");
    CPB_TRY(mlp_forward_loss(pl, L, cfg, params, source, target, eps, false, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, cfg->base.loss_scale, losses, s));
    const size_t n = (size_t)pl.B * pl.z * sizeof(float);
    if (mean) CPB_CUDA(cudaMemcpyAsync(mean, pl.heads, n, cudaMemcpyDeviceToDevice, s));
    if (logvar) CPB_CUDA(cudaMemcpyAsync(logvar, pl.heads + (long long)pl.B * pl.z, n, cudaMemcpyDeviceToDevice, s));
    if (z) CPB_CUDA(cudaMemcpyAsync(z, pl.zbuf, n, cudaMemcpyDeviceToDevice, s));
    if (reconstruction) CPB_TRY(launch_sigmoid(pl.logits, reconstruction, (long long)pl.B * pl.OUT, s));
    return CPB_OK;
}

int32_t cpb_mlpvae_loss_grad(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target, const float* eps,
                             float* grads, float* losses, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_TRAIN);
    CPB_REQUIRE(params && source && target && grads && losses, "mlp loss_grad: NULL pointer");
    CPB_TRY(mlp_forward_loss(pl, L, cfg, params, source, target, eps, true, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, cfg->base.loss_scale, losses, s));
    return mlp_backward(pl, L, cfg, params, eps, grads, s);
}

}  // extern "C"
