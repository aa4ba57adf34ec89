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

// 0: fp32 SIMT everywhere; 1: 3xTF32 wgmma for the dense conv/deconv layers; 2: the same layers as ONE TF32 wgmma
// pass with operands rounded to nearest (not fp32-accurate: up to 2^-10 relative error per product)
int g_math_mode = 1;
static int tc_passes() { return g_math_mode == 2 ? 1 : 3; }
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

// ---------------------------------------------------------------------------------------------
// geometry (layer table SURVEY appendix A.1).  The source frame is H x W x 3 (80x160 by default, reference
// vae_common.py:18-20); the encoder's four 4x4 stride-2 VALID convolutions give H1 = H/2 - 1, H2 = H/4 - 2, H3 = H/8 - 2,
// H4 = H/16 - 2 (the same in W), and the decoder (dense1 -> [H4, W4, 256] -> deconvolutions with kernels 4, 4, 5, 4)
// maps H4 back to exactly H only when H is a multiple of 16 (reference vae/models.py:265 asserts it).
// ---------------------------------------------------------------------------------------------
struct Side { int H, W, C; };
constexpr int C1 = 32, C4 = 256;
constexpr int kSideChannels[5] = {3, C1, 64, 128, C4};
constexpr int kDefaultH = 80, kDefaultW = 160;
constexpr int kMinFrameSide = 48;                       // the encoder then ends on one pixel (H4 = 1)
struct Geo {
    Side s[5];      // s[0]: the source frame; s[i]: conv i's output (conv1 [39,79,32] ... conv4 [3,8,256] at 80x160)
    int FEAT;       // H4 * W4 * 256: the flattened encoder output, dense1's width (6144 at 80x160)
    int64_t NPIX;   // H * W
    FrameGeo frame() const { return frame_geo(s[0].H, s[0].W); }
};
static Geo make_geo(int H, int W) {
    Geo g;
    g.s[0] = Side{H, W, kSideChannels[0]};
    for (int i = 1; i < 5; ++i) g.s[i] = Side{(g.s[i - 1].H - 4) / 2 + 1, (g.s[i - 1].W - 4) / 2 + 1, kSideChannels[i]};
    g.FEAT = g.s[4].H * g.s[4].W * C4;
    g.NPIX = (int64_t)H * W;
    return g;
}
static bool frame_side_ok(int v) { return v >= kMinFrameSide && v <= kMaxFrameSide && v % 16 == 0; }
#define CPB_FRAME_RULE "frame %dx%d: height and width must each be a multiple of 16 in [48, 512]"
// The MlpVAE keeps the reference's 80x160 input (its own frame size is a separate spec)
constexpr int kMlpNpix = kDefaultH * kDefaultW;

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

// ---------------------------------------------------------------------------------------------
// workspace plan
// ---------------------------------------------------------------------------------------------
constexpr int kTcLayerCount = 6;
struct TcW { int64_t f_hi, f_lo, t_hi, t_lo; };   // gather-form / quad-scatter-form K-major hi/lo copies of one kernel
struct Relayout {
    int64_t T[kTcLayerCount];       // scatter-form kernels [kh][kw][cs][cb] of the SIMT tap-GEMM, by TC_* slot
    int64_t dense1T, headsT, conv1P, deconv4P;
    TcW tc[kTcLayerCount];          // by TC_* slot
    // z < z_pad only (empty otherwise): zero-padded copies of the z-sized weights, [2][6144][z_pad], [2][z_pad], [z_pad][6144]
    int64_t headsP, headsBP, dense1P;
    int64_t total;
};
enum { TC_CONV2, TC_CONV3, TC_CONV4, TC_DECONV1, TC_DECONV2, TC_DECONV3 };

// Inside the library the latent has z_pad = 64 * ceil(z / 64) columns: the heads and dense1 then run the shapes of a
// multiple-of-64 model (the k-split tap-GEMM needs N % 64 == 0).  The padded columns hold zeros.
static int z_pad(int z) { return (int)align_up(z, 64); }

struct VaePlan {
    int B, ct, z, zp, mode;     // zp = z_pad(z): row pitch of every latent buffer (heads, zbuf, gz, gheads, ksplit)
    Geo g;
    Relayout rl;
    float *relayout, *xp, *yp, *a1, *a2, *a3, *a4, *heads, *zbuf, *kl_rows, *kl_active, *frame_loss;
    float *d1, *b1, *b2, *b3, *logits_p;
    float *gA, *gB, *gz, *gheads, *partial, *colsum;
    float* cs_edge;     // per-CTA column sums of deconv4's data gradient (edge_gather), [edge_gather_blocks(B, g)][32]
    float* frame_dsum;  // per-frame channel sums of d loss / d logits, [B][4]
    float* ksplit;      // partial results of the k-split dense layers: kMaxKSplit x [2, B, z_pad]
    int64_t bytes;
};

// ---------------------------------------------------------------------------------------------
// The six stride-2 layers on the tap-GEMM, in the big/small notation of DESIGN §2 (kernel [k][k][Cb][Cs]): a conv maps its
// big side to its small side, a deconv the other way round.  The gather form of a pass reads the big side and the kernel
// as stored (TF32 image TcW::f_*), the scatter form the small side and Relayout::T (TF32 quad image TcW::t_*).  The form
// rule (uses_scatter): a conv's forward pass runs the gather form and its data gradient the scatter form; a deconv's the
// other way round.
// ---------------------------------------------------------------------------------------------
struct TcLayer {
    const char *fwd, *wgrad, *dgrad;        // profile labels of the three passes; dgrad also names the backward stop
    int kernel, bias, slot;                 // VaeTensor, VaeTensor, TC_*
    bool deconv;
    int k;
    int big, small;                         // their sides: Geo::s indices
    float *VaePlan::*in, *VaePlan::*out;    // the forward pass's input and output activation
    bool edge;                              // the bias gradient comes from the column sums edge_gather left in cs_edge
    bool linear;                            // the input has no ReLU: the data gradient is not masked
};

#define CPB_TC_LABELS(name) name ".fwd", name ".wgrad", name ".dgrad"
static const TcLayer kTcLayers[kTcLayerCount] = {
    //                         kernel       bias         slot        deconv k  big      small    in            out           edge   linear
    {CPB_TC_LABELS("conv2"),   T_CONV2_K,   T_CONV2_B,   TC_CONV2,   false, 4, 1,   2,     &VaePlan::a1, &VaePlan::a2, false, false},
    {CPB_TC_LABELS("conv3"),   T_CONV3_K,   T_CONV3_B,   TC_CONV3,   false, 4, 2,   3,     &VaePlan::a2, &VaePlan::a3, false, false},
    {CPB_TC_LABELS("conv4"),   T_CONV4_K,   T_CONV4_B,   TC_CONV4,   false, 4, 3,   4,     &VaePlan::a3, &VaePlan::a4, false, false},
    // d1, dense1's output, is linear
    {CPB_TC_LABELS("deconv1"), T_DECONV1_K, T_DECONV1_B, TC_DECONV1, true,  4, 3,   4,     &VaePlan::d1, &VaePlan::b1, false, true},
    {CPB_TC_LABELS("deconv2"), T_DECONV2_K, T_DECONV2_B, TC_DECONV2, true,  4, 2,   3,     &VaePlan::b1, &VaePlan::b2, false, false},
    // deconv4's data gradient (edge_gather) leaves the column sums of deconv3's output gradient in cs_edge
    {CPB_TC_LABELS("deconv3"), T_DECONV3_K, T_DECONV3_B, TC_DECONV3, true,  5, 1,   2,     &VaePlan::b2, &VaePlan::b3, true,  false},
};

static bool uses_scatter(const TcLayer& l, bool dgrad) { return l.deconv != dgrad; }

// The largest batch the tensor-core kernels address with their 32-bit offsets (tc_offsets_fit) at geometry g: every
// table layer's big and small side as a tc_tapgemm source / destination and as tc_wgrad's big operand
static int64_t tc_batch_limit(const Geo& g) {
    int64_t limit = INT64_MAX;
    for (const TcLayer& l : kTcLayers)
        for (int side : {l.big, l.small}) {
            const Side& d = g.s[side];
            limit = std::min<int64_t>(limit, tc_max_batch((int64_t)d.H * d.W * d.C));
        }
    return limit;
}

static VaeLayout make_layout(int ct, int z, const Geo& g) {
    const int FEAT = g.FEAT;
    VaeLayout L;
    set_shape(L, T_CONV1_K, 4, 4, 3, C1);    set_shape(L, T_CONV1_B, C1);
    for (const TcLayer& l : kTcLayers) {
        set_shape(L, l.kernel, l.k, l.k, kSideChannels[l.big], kSideChannels[l.small]);
        set_shape(L, l.bias, kSideChannels[l.deconv ? l.big : l.small]);
    }
    set_shape(L, T_MEAN_K, FEAT, z);         set_shape(L, T_MEAN_B, z);
    set_shape(L, T_LOGVAR_K, FEAT, z);       set_shape(L, T_LOGVAR_B, z);
    set_shape(L, T_DENSE1_K, z, FEAT);       set_shape(L, T_DENSE1_B, FEAT);
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

static Relayout make_relayout(int z, const Geo& g) {
    const int FEAT = g.FEAT;
    const int zp = z_pad(z);
    const bool padded = zp != z;
    Relayout r;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
    for (const TcLayer& l : kTcLayers) r.T[l.slot] = take((int64_t)l.k * l.k * kSideChannels[l.big] * kSideChannels[l.small]);
    r.dense1T = take((int64_t)zp * FEAT);
    r.headsT = take(2LL * zp * FEAT);
    r.conv1P = take(16LL * 4 * C1);
    r.deconv4P = take(16LL * 4 * C1);
    for (const TcLayer& l : kTcLayers) {
        const int64_t cb = kSideChannels[l.big], cs = kSideChannels[l.small];
        const int64_t n = (int64_t)l.k * l.k * cb * cs, win = (l.k + 1) / 2;
        TcW& w = r.tc[l.slot];
        w.f_hi = take(n); w.f_lo = take(n);
        w.t_hi = take(win * win * 4 * cb * cs); w.t_lo = take(win * win * 4 * cb * cs);
    }
    r.headsP = take(padded ? 2LL * FEAT * zp : 0);
    r.headsBP = take(padded ? 2LL * zp : 0);
    r.dense1P = take(padded ? (int64_t)zp * FEAT : 0);
    r.total = o;
    return r;
}

static int64_t max_partial_floats(int B, int zp, const Geo& g) {
    const int FEAT = g.FEAT;
    // the tensor-core weight gradient runs ONE wave of (i-tile, j-tile, split) CTAs with 128 x BN <= 128 x 64 tiles
    int64_t best = std::max<int64_t>((int64_t)edge_wgrad_ctas(B, g.frame()) * 48 * C1, (int64_t)kTcWaveCtas * 128 * 64);
    auto fit = [&](int I, int J, long long M) {
        best = std::max<int64_t>(best, (int64_t)wgrad_pick_splits(I, J, M) * I * J);
        best = std::max<int64_t>(best, (int64_t)tc_wgrad_pick_splits(I, J, M) * I * J);
    };
    fit(64, C1, (long long)B * g.s[1].H * g.s[1].W);        // conv1 / deconv4 (padded to 4 channels)
    for (const TcLayer& l : kTcLayers) {
        const Side &big = g.s[l.big], &small = g.s[l.small];
        fit(l.k * l.k * big.C, small.C, (long long)B * small.H * small.W);
    }
    fit(FEAT, zp, B);                           // heads
    fit(zp, FEAT, B);                           // dense1
    return best;
}

static VaePlan make_plan(void* ws, int64_t ws_bytes, int B, int ct, int z, int mode, const Geo& g) {
    const int64_t FEAT = g.FEAT, NPIX = g.NPIX;
    const int64_t H1 = g.s[1].H, W1 = g.s[1].W, H2 = g.s[2].H, W2 = g.s[2].W, H3 = g.s[3].H, W3 = g.s[3].W;
    const int64_t C2 = g.s[2].C, C3 = g.s[3].C;
    VaePlan p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.ct = ct; p.z = z; p.zp = z_pad(z); p.mode = mode; p.g = g;
    p.rl = make_relayout(z, g);
    const int64_t zp = p.zp;
    Arena a(ws, ws_bytes);
    const int64_t b = B;
    p.relayout = a.take<float>(p.rl.total);
    p.xp = a.take<float>(b * NPIX * 4);
    p.a1 = a.take<float>(b * H1 * W1 * C1);
    p.a2 = a.take<float>(b * H2 * W2 * C2);
    p.a3 = a.take<float>(b * H3 * W3 * C3);
    p.a4 = a.take<float>(b * FEAT);
    p.heads = a.take<float>(2 * b * zp);
    p.ksplit = a.take<float>((int64_t)kMaxKSplit * 2 * b * zp);
    if (mode >= CPB_WS_FORWARD) {
        p.yp = a.take<float>(b * NPIX * 4);
        p.zbuf = a.take<float>(b * zp);
        p.kl_rows = a.take<float>(b);
        p.kl_active = a.take<float>(b);
        p.frame_loss = a.take<float>(b);
        p.d1 = a.take<float>(b * FEAT);
        p.b1 = a.take<float>(b * H3 * W3 * C3);
        p.b2 = a.take<float>(b * H2 * W2 * C2);
        p.b3 = a.take<float>(b * H1 * W1 * C1);
        p.logits_p = a.take<float>(b * NPIX * 4);
    }
    if (mode >= CPB_WS_TRAIN) {
        p.gA = a.take<float>(b * H1 * W1 * C1);
        p.gB = a.take<float>(b * H1 * W1 * C1);
        p.gz = a.take<float>(b * zp);
        p.gheads = a.take<float>(2 * b * zp);
        p.partial = a.take<float>(max_partial_floats(B, p.zp, g));
        p.colsum = a.take<float>(colsum_scratch_floats(b * NPIX, 4) + colsum_scratch_floats(b * H1 * W1, C1) +
                                 colsum_scratch_floats(b, (int)FEAT));
        p.cs_edge = a.take<float>(edge_gather_blocks(B, g.frame()) * C1);
        p.frame_dsum = a.take<float>(b * 4);
    }
    p.bytes = a.off;
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

static int32_t tg(const char* label, const TapGemmParams& p, cudaStream_t s, int scatter_k = 0) {
    ProfScope prof(label, s);
    if (g_math_mode >= 1 && p.wk_hi != nullptr) {
        TapGemmParams q = scatter_k > 0 ? quad_from_scatter(p, scatter_k) : p;
        q.debug = tc_debug_flags();
        q.passes = tc_passes();
        if (tc_tapgemm_supported(q)) return launch_tc_tapgemm(q, s);
    }
    return launch_tapgemm(p, s);
}

// out[k][k][Cb][Cs] = the weight gradient of table layer l from its big-side and small-side operands
static int32_t run_wgrad(const TcLayer& l, const Geo& g, const float* big, const float* small, int B, float* partial, float* out,
                         cudaStream_t s) {
    ProfScope prof(l.wgrad, s);
    const Side &bs = g.s[l.big], &ss = g.s[l.small];
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = big; w.small = small; w.partial = partial;
    w.batch = B; w.Wb = bs.W; w.big_pitch = bs.C; w.big_img = (long long)bs.H * bs.W * bs.C;
    w.Ho = ss.H; w.Wo = ss.W; w.sstride = 2;
    w.ntaps = l.k; w.run = l.k * bs.C;
    for (int kh = 0; kh < l.k; ++kh) w.tap_off[kh] = (long long)kh * bs.W * bs.C;
    w.I = l.k * l.k * bs.C; w.J = ss.C;
    const long long M = (long long)B * ss.H * ss.W;
    if (g_math_mode >= 1 && tc_wgrad_supported(w.I, w.J, w.run)) {
        w.passes = tc_passes();
        w.splits = tc_wgrad_pick_splits(w.I, w.J, M);
        w.m_per_split = align_up((M + w.splits - 1) / w.splits, 32);
        CPB_TRY(launch_tc_wgrad(w, s));
    } else {
        w.splits = wgrad_pick_splits(w.I, w.J, M);
        w.m_per_split = align_up((M + w.splits - 1) / w.splits, 16);
        CPB_TRY(launch_wgrad(w, s));
    }
    return launch_reduce_partials(partial, w.splits, w.I, w.J, w.I, w.I, w.J, out, s);
}

// out[k_real][j_real] = x[B, K]^T g[B, J], dropping the padded rows k >= k_real and columns j >= j_real
static int32_t run_dense_wgrad(const char* label, const float* x, int K, int k_real, const float* g, int B, int J, int j_real,
                               float* partial, float* out, cudaStream_t s) {
    ProfScope prof(label, s);
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = x; w.small = g; w.partial = partial;
    w.batch = B; w.Wb = 1; w.big_pitch = K; w.big_img = K; w.Ho = w.Wo = 1; w.sstride = 1;
    w.ntaps = 1; w.run = K; w.tap_off[0] = 0; w.I = K; w.J = J;
    w.splits = wgrad_pick_splits(w.I, w.J, B);
    w.m_per_split = align_up(((long long)B + w.splits - 1) / w.splits, 16);
    CPB_TRY(launch_wgrad(w, s));
    return launch_reduce_partials(partial, w.splits, w.I, w.J, K, k_real, j_real, out, s);
}

// ---------------------------------------------------------------------------------------------
// passes
// ---------------------------------------------------------------------------------------------
// multiples of 4: every [B, z] row that crosses the ABI starts 16-byte aligned, so the pitch changes move float4
static bool z_ok(int z) { return z >= 4 && z % 4 == 0 && z <= 1024; }
#define CPB_Z_RULE "z_dim=%d must be a multiple of 4 in [4,1024]"

static int32_t check_cfg(const cpb_vae_config* cfg) {
    CPB_REQUIRE(cfg != nullptr, "cfg is NULL");
    CPB_REQUIRE(cfg->batch >= 1 && cfg->batch <= (1 << 20), "batch=%d out of range", cfg->batch);
    CPB_REQUIRE(cfg->target_channels == 1 || cfg->target_channels == 3, "target_channels must be 1 or 3, got %d", cfg->target_channels);
    CPB_REQUIRE(z_ok(cfg->z_dim), CPB_Z_RULE, cfg->z_dim);
    CPB_REQUIRE(cfg->loss_type >= 0 && cfg->loss_type <= 2, "unknown loss_type %d", cfg->loss_type);
    CPB_REQUIRE(cfg->source_dtype == CPB_FRAME_F32 || cfg->source_dtype == CPB_FRAME_U8, "bad source_dtype");
    CPB_REQUIRE(cfg->target_dtype == CPB_FRAME_F32 || cfg->target_dtype == CPB_FRAME_U8, "bad target_dtype");
    return CPB_OK;
}

static int32_t check_frame(int H, int W) {
    CPB_REQUIRE(frame_side_ok(H) && frame_side_ok(W), CPB_FRAME_RULE, H, W);
    return CPB_OK;
}

static int32_t check_spec(const cpb_vae_spec* sp) {
    CPB_REQUIRE(sp != nullptr, "cfg is NULL");
    CPB_TRY(check_cfg(&sp->base));
    return check_frame(sp->height, sp->width);
}

// Math modes 1 and 2 run the table layers on the tensor-core kernels, whose 32-bit offsets bound the batch
// (tc_batch_limit): a larger batch is refused here, before the call launches anything.  The fp32 SIMT kernels of mode 0
// index with 64-bit offsets and take every batch check_cfg accepts.
static int32_t check_batch_bound(const cpb_vae_spec* sp, const Geo& g) {
    const int64_t limit = tc_batch_limit(g);
    if (g_math_mode == 0 || sp->base.batch <= limit) return CPB_OK;
    set_error("batch=%d is above %lld, the largest batch the tensor-core kernels (math modes 1 and 2) take at frame %dx%d",
              sp->base.batch, (long long)limit, sp->height, sp->width);
    return CPB_ERR_UNSUPPORTED;
}

static void add_relayout(RelayoutTable& t, int64_t src, int64_t dst, int taps, int rows, int cols, int mode,
                         int rows_pad, int cols_pad) {
    RelayoutJob& j = t.jobs[t.njobs++];
    j.src_off = src; j.dst_off = dst; j.taps = taps; j.rows = rows; j.cols = cols; j.mode = mode;
    j.rows_pad = rows_pad; j.cols_pad = cols_pad;
    j.count = (long long)taps * rows_pad * cols_pad;
    t.total += j.count;
}

// The latent block both VAEs share: the two heads (mean, logstd_sq) over a [B, K] layer, z_pad-column latent rows
struct Latent {
    int B, K, z, zp;
    const int64_t* off;     // the VAE's parameter offsets
    int mean;               // tensor index of mean/kernel; mean/bias, logstd_sqare/kernel and logstd_sqare/bias follow it
};

// Both heads as one y-batched dense problem over x [B, K]: heads[0] = mean, heads[1] = logstd_sq.  The weights are the
// parameters (both kernels, and both biases, are adjacent) when z == z_pad, the zero-padded wp and bp otherwise.
static TapGemmParams heads_fwd_problem(const Latent& h, const float* params, const float* x, const float* wp, const float* bp,
                                       float* heads) {
    const bool padded = h.zp != h.z;
    TapGemmParams p = dense_problem(x, h.B, h.K, padded ? wp : params + h.off[h.mean], h.zp,
                                    padded ? bp : params + h.off[h.mean + 1], nullptr, heads, 0);
    p.ybatch = 2;
    p.w_ystride = padded ? (long long)h.K * h.zp : h.off[h.mean + 2] - h.off[h.mean];
    p.bias_ystride = padded ? h.zp : h.off[h.mean + 3] - h.off[h.mean + 1];
    p.dst_ystride = (long long)h.B * h.zp;
    return p;
}

// The heads' weight and bias gradients from gheads [2][B][z_pad], then their data gradient into gx = g(x pre-activation)
// = gmean Wm^T + glogvar Wl^T with wt = both kernels transposed, [2][z_pad][K].  dgrad_label may be null: no profile scope.
static int32_t heads_backward(const Latent& h, const char* wgrad_label, const char* dgrad_label, const float* x, const float* gheads,
                              const float* wt, float* gx, float* partial, float* cs, float* grads, cudaStream_t s) {
    const long long glogvar = (long long)h.B * h.zp;
    CPB_TRY(run_dense_wgrad(wgrad_label, x, h.K, h.K, gheads, h.B, h.zp, h.z, partial, grads + h.off[h.mean], s));
    CPB_TRY(run_dense_wgrad(wgrad_label, x, h.K, h.K, gheads + glogvar, h.B, h.zp, h.z, partial, grads + h.off[h.mean + 2], s));
    CPB_TRY(launch_colsum(gheads, h.B, h.zp, h.z, grads + h.off[h.mean + 1], cs, s));
    CPB_TRY(launch_colsum(gheads + glogvar, h.B, h.zp, h.z, grads + h.off[h.mean + 3], cs, s));
    TapGemmParams p = dense_problem(gheads, h.B, h.zp, wt, h.K, nullptr, x, gx, 0);
    p.cls[0].ntaps = 2;
    p.cls[0].taps[1].dy = p.cls[0].taps[1].dx = 0;
    p.cls[0].taps[1].src_off = glogvar;
    p.cls[0].taps[1].w_off = (long long)h.zp * h.K;
    if (dgrad_label == nullptr) return launch_tapgemm(p, s);
    ProfScope prof(dgrad_label, s);
    return launch_tapgemm(p, s);
}

// z < z_pad: the zero-padded copies of the z-sized weights -- `heads`: both kernels [2][K][z_pad] at wp, both biases
// [2][z_pad] at bp; `dec`: the first decoder layer's kernel [z][N] at parameter offset dec_off, as [z_pad][N] at dp
static void add_z_padding(RelayoutTable& t, const Latent& h, bool heads, int64_t wp, int64_t bp, bool dec, int64_t dec_off,
                          int N, int64_t dp) {
    if (h.zp == h.z) return;
    if (heads) {
        add_relayout(t, h.off[h.mean], wp, 2, h.K, h.z, 1, h.K, h.zp);
        add_relayout(t, h.off[h.mean + 1], bp, 1, 1, h.z, 1, 1, h.zp);
        add_relayout(t, h.off[h.mean + 3], bp + h.zp, 1, 1, h.z, 1, 1, h.zp);
    }
    if (dec) add_relayout(t, dec_off, dp, 1, h.z, N, 1, h.zp, N);
}

// An rgb target that is the source itself (vae/train_vae.py:75) is read from the source's prepared, range-checked copy
static bool target_is_source(const cpb_vae_config* c, const void* source, const void* target) {
    return target == source && c->target_channels == 3 && c->target_dtype == c->source_dtype &&
           (c->target_dtype == CPB_FRAME_F32 || c->target_u8_scale == 1.f / 255.f);
}

// [B, z_pad] latent rows of the workspace -> the caller's [B, z] rows of mean, logvar (heads) and z (zbuf), where given
static int32_t copy_latents_out(const float* heads, const float* zbuf, int B, int z, int zp, float* mean, float* logvar,
                                float* zout, cudaStream_t s) {
    const float* src[3] = {heads, heads + (long long)B * zp, zbuf};
    float* dst[3] = {mean, logvar, zout};
    for (int i = 0; i < 3; ++i) {
        if (dst[i] == nullptr) continue;
        if (zp == z)
            CPB_CUDA(cudaMemcpyAsync(dst[i], src[i], (size_t)B * z * sizeof(float), cudaMemcpyDeviceToDevice, s));
        else
            CPB_TRY(launch_pitch_copy(src[i], zp, dst[i], z, B, s));
    }
    return CPB_OK;
}

static int32_t relayout_weights(const VaePlan& pl, const VaeLayout& L, const float* params, bool encoder, bool decoder,
                                bool backward, cudaStream_t s) {
    const int FEAT = pl.g.FEAT;
    RelayoutTable t;
    memset(&t, 0, sizeof(t));
    TcWeightTable w;
    memset(&w, 0, sizeof(w));
    const int round_nearest = tc_passes() == 1 ? 1 : 0;
    auto addw = [&](const TcLayer& l, bool scatter) {
        const TcW& at = pl.rl.tc[l.slot];
        const int win = (l.k + 1) / 2;
        const int cb = kSideChannels[l.big], cs = kSideChannels[l.small];
        TcWeightJob& j = w.jobs[w.njobs++];
        j.src_off = L.off[l.kernel]; j.round_nearest = round_nearest;
        j.mode = scatter ? 2 : 1; j.k = l.k; j.cb = cb; j.cs = cs;
        j.dst_hi = scatter ? at.t_hi : at.f_hi; j.dst_lo = scatter ? at.t_lo : at.f_lo;
        j.N = scatter ? 4 * cb : cs; j.C = scatter ? cs : l.k * cb;
        j.count = (long long)j.N * j.C * (scatter ? win * win : l.k); w.total += j.count;
    };
    // the forms of each layer that the call's passes run: the scatter form's SIMT transpose, and each form's TF32 image
    for (const TcLayer& l : kTcLayers) {
        const bool fwd = l.deconv ? decoder : encoder;
        const bool scatter = (fwd && uses_scatter(l, false)) || (backward && uses_scatter(l, true));
        const bool gather = (fwd && !uses_scatter(l, false)) || (backward && !uses_scatter(l, true));
        const int cb = kSideChannels[l.big], cs = kSideChannels[l.small];
        if (scatter) add_relayout(t, L.off[l.kernel], pl.rl.T[l.slot], l.k * l.k, cb, cs, 0, cb, cs);
        if (gather) addw(l, false);
        if (scatter) addw(l, true);
    }
    if (backward) {
        add_relayout(t, L.off[T_DENSE1_K], pl.rl.dense1T, 1, pl.z, FEAT, 0, pl.zp, FEAT);      // [6144][z_pad]
        add_relayout(t, L.off[T_MEAN_K], pl.rl.headsT, 2, FEAT, pl.z, 0, FEAT, pl.zp);        // [2][z_pad][6144]: mean and logvar kernels are adjacent
    }
    add_z_padding(t, Latent{pl.B, FEAT, pl.z, pl.zp, L.off, T_MEAN_K}, encoder, pl.rl.headsP, pl.rl.headsBP, decoder,
                  L.off[T_DENSE1_K], FEAT, pl.rl.dense1P);
    ProfScope prof("relayout_weights", s);
    CPB_TRY(launch_relayout(params, pl.relayout, t, s));
    if (g_math_mode == 0) return CPB_OK;
    return launch_tc_weights(params, pl.relayout, w, s);
}

// A table layer's forward pass (bias, ReLU) or data gradient (ReLU mask `mask`, if any) in the form uses_scatter gives:
// src is the big side and dst the small side in the gather form, the other way round in the scatter form
static int32_t run_layer_pass(const VaePlan& pl, const VaeLayout& L, const float* params, const TcLayer& l, bool dgrad,
                              const float* src, const float* mask, float* dst, cudaStream_t s) {
    const char* label = dgrad ? l.dgrad : l.fwd;
    const float* bias = dgrad ? nullptr : params + L.off[l.bias];
    const int relu = dgrad ? 0 : 1;
    const float* rl = pl.relayout;
    const TcW& w = pl.rl.tc[l.slot];
    const Side &big = pl.g.s[l.big], &small = pl.g.s[l.small];
    if (uses_scatter(l, dgrad))
        return tg(label, scatter_problem(src, pl.B, small.H, small.W, small.C, l.k, rl + pl.rl.T[l.slot], big.C, bias,
                                         mask, dst, big.H, big.W, relu, rl + w.t_hi, rl + w.t_lo), s, l.k);
    return tg(label, gather_problem(src, pl.B, big.H, big.W, big.C, l.k, params + L.off[l.kernel], small.C, bias, mask,
                                    dst, relu, rl + w.f_hi, rl + w.f_lo), s, 0);
}

static int32_t run_encoder(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                           const void* source, int32_t* flags, cudaStream_t s) {
    const int B = pl.B, FEAT = pl.g.FEAT;
    const float sscale = cfg->source_dtype == CPB_FRAME_U8 ? 1.f / 255.f : 1.f;
    { ProfScope prof("prep_frames", s);
      CPB_TRY(launch_prep_frames(source, cfg->source_dtype, sscale, 3, B * pl.g.NPIX, pl.xp, flags, 1, s)); }
    { ProfScope prof("conv1.fwd", s);
      CPB_TRY(launch_edge_gather(pl.xp, 3, params + L.off[T_CONV1_K], params + L.off[T_CONV1_B], nullptr, pl.a1, B, pl.g.frame(), s)); }
    for (int i = TC_CONV2; i <= TC_CONV4; ++i)
        CPB_TRY(run_layer_pass(pl, L, params, kTcLayers[i], false, pl.*kTcLayers[i].in, nullptr, pl.*kTcLayers[i].out, s));
    TapGemmParams p = heads_fwd_problem(Latent{B, FEAT, pl.z, pl.zp, L.off, T_MEAN_K}, params, pl.a4, pl.relayout + pl.rl.headsP,
                                        pl.relayout + pl.rl.headsBP, pl.heads);
    p.ksplit = tapgemm_pick_ksplit(B, pl.zp, 2, FEAT);
    p.kpartial = pl.ksplit; p.kpartial_stride = 2LL * B * pl.zp;
    return tg("heads.fwd", p, s);
}

// zsrc [B, z_pad] -> d1 -> b1 -> b2 -> b3 -> (logits_p and/or sigmoid)
static int32_t run_decoder(const VaePlan& pl, const VaeLayout& L, const float* params, const float* zsrc,
                           float* logits_p, float* sigm, cudaStream_t s) {
    const int B = pl.B, FEAT = pl.g.FEAT;
    const float* w1 = pl.zp != pl.z ? pl.relayout + pl.rl.dense1P : params + L.off[T_DENSE1_K];
    TapGemmParams p = dense_problem(zsrc, B, pl.zp, w1, FEAT, params + L.off[T_DENSE1_B], nullptr, pl.d1, 0);
    CPB_TRY(tg("dense1.fwd", p, s));
    for (int i = TC_DECONV1; i <= TC_DECONV3; ++i)
        CPB_TRY(run_layer_pass(pl, L, params, kTcLayers[i], false, pl.*kTcLayers[i].in, nullptr, pl.*kTcLayers[i].out, s));
    ProfScope prof("deconv4.fwd", s);
    return launch_deconv4_fwd(pl.b3, params + L.off[T_DECONV4_K], params + L.off[T_DECONV4_B], B, pl.ct, pl.g.frame(),
                              logits_p, sigm, s);
}

static int32_t run_forward_loss(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                                const void* source, const void* target, const float* eps, bool want_dlogits,
                                float* sigm, int32_t* flags, cudaStream_t s) {
    const int B = pl.B;
    CPB_TRY(run_encoder(pl, L, cfg, params, source, flags, s));
    CPB_TRY(launch_reparam(pl.heads, eps, B, pl.z, pl.zp, cfg->kl_tolerance, pl.zbuf, pl.kl_rows, pl.kl_active, s));
    CPB_TRY(run_decoder(pl, L, params, pl.zbuf, pl.logits_p, sigm, s));
    const float* yp = target_is_source(cfg, source, target) ? pl.xp : pl.yp;
    if (yp == pl.yp) {
        const float tscale = cfg->target_dtype == CPB_FRAME_U8 ? cfg->target_u8_scale : 1.f;
        CPB_TRY(launch_prep_frames(target, cfg->target_dtype, tscale, cfg->target_channels, B * pl.g.NPIX,
                                   pl.yp, flags, 2, s));
    }
    const float gscale = cfg->loss_scale / (float)B;
    { ProfScope prof("recon_loss", s);
      CPB_TRY(launch_recon_loss(pl.logits_p, yp, B, (int)pl.g.NPIX, pl.ct, cfg->loss_type, gscale, pl.frame_loss,
                                want_dlogits ? pl.logits_p : nullptr, s, want_dlogits ? pl.frame_dsum : nullptr)); }
    return CPB_OK;
}

// cpb_debug_vae_backward_stop: the layer groups of run_backward after which it may return early, in pass order.  Each
// group is the layer's weight gradient, bias gradient and data gradient; the stop comes after all three.
static const char* kBackwardStops[] = {"deconv4.dgrad", "deconv3.dgrad", "deconv2.dgrad", "deconv1.dgrad", "dense1.dgrad",
                                       "heads.dgrad", "conv4.dgrad", "conv3.dgrad"};
static const char* g_backward_stop = nullptr;    // the kBackwardStops entry run_backward stops after; null: none
#define CPB_BACKWARD_STOP(group) if (g_backward_stop != nullptr && strcmp(g_backward_stop, group) == 0) return CPB_OK

// A table layer's group of the backward pass: its weight gradient, bias gradient and data gradient.  g is the gradient at
// the layer's output (pre-activation); gin receives the one at its input, masked by the input's ReLU.
static int32_t run_layer_backward(const VaePlan& pl, const VaeLayout& L, const float* params, const TcLayer& l, const float* g,
                                  float* gin, float* grads, cudaStream_t s) {
    const float* in = pl.*l.in;
    const Side& out = pl.g.s[l.deconv ? l.big : l.small];
    CPB_TRY(run_wgrad(l, pl.g, l.deconv ? g : in, l.deconv ? in : g, pl.B, pl.partial, grads + L.off[l.kernel], s));
    if (l.edge)
        CPB_TRY(launch_colsum(pl.cs_edge, edge_gather_blocks(pl.B, pl.g.frame()), out.C, out.C, grads + L.off[l.bias], pl.colsum, s));
    else
        CPB_TRY(launch_colsum(g, (long long)pl.B * out.H * out.W, out.C, out.C, grads + L.off[l.bias], pl.colsum, s));
    return run_layer_pass(pl, L, params, l, true, g, l.linear ? nullptr : in, gin, s);
}

static int32_t run_backward(const VaePlan& pl, const VaeLayout& L, const cpb_vae_config* cfg, const float* params,
                            const float* eps, float* grads, cudaStream_t s) {
    const int B = pl.B, z = pl.z, zp = pl.zp, FEAT = pl.g.FEAT;
    const FrameGeo fg = pl.g.frame();
    float* dlog = pl.logits_p;   // overwritten in place by the loss kernel
    float* cs = pl.colsum;
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    // ---- deconv4 (padded to 4 channels on the big side)
    { ProfScope prof("deconv4.wgrad", s);
      CPB_TRY(launch_edge_wgrad(dlog, pl.ct, pl.b3, B, fg, pl.partial, s));
      CPB_TRY(launch_reduce_partials(pl.partial, edge_wgrad_ctas(B, fg), 16 * pl.ct, C1, 16 * pl.ct, 16 * pl.ct, C1,
                                     grads + L.off[T_DECONV4_K], s)); }
    // the bias gradients of the two outermost layers come out of the kernels that write their pre-activation gradients
    // (recon_loss: per-frame channel sums; edge_gather: per-CTA column sums) instead of separate passes over 0.8 + 1.6 GB
    CPB_TRY(launch_colsum(pl.frame_dsum, B, 4, pl.ct, grads + L.off[T_DECONV4_B], cs, s));
    { ProfScope prof("deconv4.dgrad", s);
      CPB_TRY(launch_edge_gather(dlog, pl.ct, params + L.off[T_DECONV4_K], nullptr, pl.b3, pl.gA, B, fg, s, pl.cs_edge)); }   // gA = g(b3 pre-activation)
    CPB_BACKWARD_STOP("deconv4.dgrad");
    // ---- deconv3, deconv2, deconv1: gA -> gB -> gA -> gB = g(d1) [B, 6144]
    float *g = pl.gA, *gin = pl.gB;
    for (int i = TC_DECONV3; i >= TC_DECONV1; --i) {
        CPB_TRY(run_layer_backward(pl, L, params, kTcLayers[i], g, gin, grads, s));
        CPB_BACKWARD_STOP(kTcLayers[i].dgrad);
        std::swap(g, gin);
    }
    // ---- dense1
    CPB_TRY(run_dense_wgrad("dense1.wgrad", pl.zbuf, zp, z, pl.gB, B, FEAT, FEAT, pl.partial, grads + L.off[T_DENSE1_K], s));
    CPB_TRY(launch_colsum(pl.gB, B, FEAT, FEAT, grads + L.off[T_DENSE1_B], cs, s));
    TapGemmParams p = dense_problem(pl.gB, B, FEAT, pl.relayout + pl.rl.dense1T, zp, nullptr, nullptr, pl.gz, 0);
    p.ksplit = tapgemm_pick_ksplit(B, zp, 1, FEAT);
    p.kpartial = pl.ksplit; p.kpartial_stride = (long long)B * zp;
    CPB_TRY(tg("dense1.dgrad", p, s));
    CPB_BACKWARD_STOP("dense1.dgrad");
    // ---- sampling + KL
    CPB_TRY(launch_reparam_bwd(pl.heads, eps, pl.gz, pl.kl_active, B, z, zp, cfg->beta * cfg->loss_scale / (float)B,
                               pl.gheads, s));
    // ---- heads: gA = g(a4 pre-activation)
    CPB_TRY(heads_backward(Latent{B, FEAT, z, zp, L.off, T_MEAN_K}, "heads.wgrad", "heads.dgrad", pl.a4, pl.gheads,
                           pl.relayout + pl.rl.headsT, pl.gA, pl.partial, cs, grads, s));
    CPB_BACKWARD_STOP("heads.dgrad");
    // ---- conv4 (from the heads' data gradient in gA), conv3, conv2: gA -> gB -> gA -> gB = g(a1)
    g = pl.gA;
    gin = pl.gB;
    for (int i = TC_CONV4; i >= TC_CONV2; --i) {
        CPB_TRY(run_layer_backward(pl, L, params, kTcLayers[i], g, gin, grads, s));
        CPB_BACKWARD_STOP(kTcLayers[i].dgrad);
        std::swap(g, gin);
    }
    // ---- conv1 (its input gradient is never used: the reference computes and discards it)
    { ProfScope prof("conv1.wgrad", s);
      CPB_TRY(launch_edge_wgrad(pl.xp, 3, pl.gB, B, fg, pl.partial, s));
      CPB_TRY(launch_reduce_partials(pl.partial, edge_wgrad_ctas(B, fg), 48, C1, 48, 48, C1, grads + L.off[T_CONV1_K], s)); }
    CPB_TRY(launch_colsum(pl.gB, (long long)B * fg.H1 * fg.W1, C1, C1, grads + L.off[T_CONV1_B], cs, s));
    return CPB_OK;
}


// =============================================================================================
// MlpVAE (reference vae/models.py:271-299, build_mlp): flatten -> one dense relu layer per encoder size -> [mean |
// logstd_sq] -> sample -> one dense relu layer per decoder size -> the output layer, dense 12800*Ct -> logits.  Same loss /
// sampling / Adam kernels as the ConvVAE; the layers run on the fp32 SIMT tap-GEMM (dense form) and the SIMT
// weight-gradient kernel, except in math mode 2: there the five frame-wide products -- the first encoder layer's forward
// and weight gradient, the output layer's forward, data gradient and weight gradient -- run as ONE TF32 wgmma pass with
// both operands rounded to nearest (the forward passes and the data gradient on the tensor-core tap-GEMM, k-split where
// they reduce over a frame, the weight gradients on tc_wgrad).  Profile labels call the output layer "dec2" at every
// depth (its name in the default two-per-side model).
// =============================================================================================
constexpr int kMlpMaxLayers = 8;                                  // hidden layers per side
constexpr int kMlpMaxTensors = 2 * (2 * kMlpMaxLayers + 3);

// Tensor indices in TF creation order: encoder layer i {kernel, bias} at 2i, mean at 2L, logstd_sqare at 2L + 2, decoder
// layer j at 2L + 4 + 2j (j = M: the output layer); a bias follows its kernel.
struct MlpLayout {
    int nenc, ndec, n;
    int64_t off[kMlpMaxTensors], size[kMlpMaxTensors];
    int32_t shape[kMlpMaxTensors][2];
    int64_t total;
    int enc(int i) const { return 2 * i; }
    int mean() const { return 2 * nenc; }
    int logvar() const { return 2 * nenc + 2; }
    int dec(int j) const { return 2 * nenc + 4 + 2 * j; }
};

// The reference's tf.layers names: build_mlp numbers the dense layers of a scope dense, dense_1, dense_2, ...
static const char* mlp_tensor_name(int nenc, int ndec, int i) {
    static const char* heads[4] = {"mean/kernel", "mean/bias", "logstd_sqare/kernel", "logstd_sqare/bias"};
    static char names[2][kMlpMaxLayers + 1][2][32];
    static const bool ready = [] {
        for (int d = 0; d < 2; ++d)
            for (int l = 0; l <= kMlpMaxLayers; ++l)
                for (int b = 0; b < 2; ++b) {
                    char suffix[8] = "";
                    if (l) snprintf(suffix, sizeof(suffix), "_%d", l);
                    snprintf(names[d][l][b], sizeof(names[d][l][b]), "%s/dense%s/%s", d ? "decoder" : "encoder", suffix,
                             b ? "bias" : "kernel");
                }
        return true;
    }();
    (void)ready;
    if (i < 0 || i >= 2 * (nenc + ndec + 3)) return nullptr;
    if (i < 2 * nenc) return names[0][i / 2][i % 2];
    if (i < 2 * nenc + 4) return heads[i - 2 * nenc];
    return names[1][(i - 2 * nenc - 4) / 2][i % 2];
}

static int32_t check_mlp_spec(const cpb_mlpvae_spec* c) {
    CPB_REQUIRE(c != nullptr, "mlp spec is NULL");
    CPB_TRY(check_cfg(&c->base));
    // an empty side would make the y-batched heads or the first decoder layer reductions over a whole frame
    CPB_REQUIRE(c->num_encoder >= 1 && c->num_encoder <= kMlpMaxLayers && c->num_decoder >= 1 && c->num_decoder <= kMlpMaxLayers,
                "MlpVAE needs 1 to %d hidden layers per side (encoder_sizes / decoder_sizes), got %d and %d", kMlpMaxLayers,
                c->num_encoder, c->num_decoder);
    for (int i = 0; i < c->num_encoder + c->num_decoder; ++i) {
        const int v = i < c->num_encoder ? c->encoder_sizes[i] : c->decoder_sizes[i - c->num_encoder];
        CPB_REQUIRE(v >= 32 && v % 32 == 0 && v <= 8192, "MlpVAE hidden sizes must be multiples of 32 in [32, 8192], got %d", v);
    }
    return CPB_OK;
}

static MlpLayout make_mlp_layout(const cpb_mlpvae_spec* c) {
    const int IN = kMlpNpix * 3, OUT = kMlpNpix * c->base.target_channels, z = c->base.z_dim;
    MlpLayout L;
    L.nenc = c->num_encoder; L.ndec = c->num_decoder; L.n = 2 * (L.nenc + L.ndec + 3);
    auto dense = [&](int t, int in, int out) {       // kernel [in, out] at t, bias [out] at t + 1
        L.shape[t][0] = in; L.shape[t][1] = out; L.size[t] = (int64_t)in * out;
        L.shape[t + 1][0] = out; L.shape[t + 1][1] = 0; L.size[t + 1] = out;
    };
    for (int i = 0; i < L.nenc; ++i) dense(L.enc(i), i ? c->encoder_sizes[i - 1] : IN, c->encoder_sizes[i]);
    const int top = c->encoder_sizes[L.nenc - 1];
    dense(L.mean(), top, z);
    dense(L.logvar(), top, z);
    for (int j = 0; j <= L.ndec; ++j) dense(L.dec(j), j ? c->decoder_sizes[j - 1] : z, j < L.ndec ? c->decoder_sizes[j] : OUT);
    // storage: creation order, except that the two head kernels (and biases) are adjacent: both heads run as one
    // y-batched dense problem
    int order[kMlpMaxTensors], n = 0;
    for (int t = 0; t < L.mean(); ++t) order[n++] = t;
    for (int t : {L.mean(), L.logvar(), L.mean() + 1, L.logvar() + 1}) order[n++] = t;
    for (int t = L.dec(0); t < L.n; ++t) order[n++] = t;
    int64_t o = 0;
    for (int i = 0; i < L.n; ++i) { L.off[order[i]] = o; o += align_up(L.size[order[i]], 64); }
    L.total = o;
    return L;
}

struct MlpPlan {
    int B, IN, OUT, z, zp;                   // zp = z_pad(z), the row pitch of the latent buffers (as in VaePlan)
    int nenc, ndec, enc[kMlpMaxLayers], dec[kMlpMaxLayers];
    float *x, *y, *h[kMlpMaxLayers], *heads, *zbuf, *kl_rows, *kl_active, *frame_loss, *g[kMlpMaxLayers], *logits;
    float *ga, *gb, *gz, *gheads, *partial, *colsum, *wT, *ksplit;
    // float offsets of the transposed kernels inside wT: encoder layers 1.. (tEnc[0] unused), the heads, decoder layers
    // 0..M (tDec[M]: the output layer)
    int64_t tEnc[kMlpMaxLayers], tHeads, tDec[kMlpMaxLayers + 1];
    float* wP;                               // z < z_pad only: zero-padded heads [2][top][z_pad], biases [2][z_pad], decoder/dense [z_pad][dec0]
    int64_t pHeads, pHeadsB, pD1;
    // math mode 2 only (tc): TF32 weight images of the frame-wide layers inside wTc -- the first encoder layer K-major
    // [enc0][IN] (every mode), the output layer K-major [OUT][dec_last] (forward and train) and as stored [dec_last][OUT]
    // (train, data gradient) -- and tcScratch for the k-split partials and the tensor-core weight-gradient partials
    bool tc;
    float *wTc, *tcScratch;
    int64_t iE1, iD3f, iD3t;
    int64_t bytes;
    int top() const { return enc[nenc - 1]; }
    int last() const { return dec[ndec - 1]; }
};

// The tensor-core kernels address a frame-wide operand with 32-bit offsets (B * 38 400 < 2^31, i.e. B <= 55 923):
// a larger batch runs the five products on the fp32 SIMT kernels in every mode.
static bool mlp_tc_batch_ok(int64_t b, int in) { return b * in < (1LL << 31); }

static int64_t mlp_tc_scratch_floats(const MlpPlan& p, int mode) {
    const int64_t b = p.B;
    int64_t n = (int64_t)tc_tapgemm_pick_ksplit(p.IN) * b * p.enc[0];                              // first encoder layer fwd
    if (mode >= CPB_WS_TRAIN) {
        n = std::max<int64_t>(n, (int64_t)tc_tapgemm_pick_ksplit(p.OUT) * b * p.last());           // output layer dgrad
        n = std::max<int64_t>(n, (int64_t)tc_wgrad_pick_splits(p.IN, p.enc[0], b) * p.IN * p.enc[0]);
        n = std::max<int64_t>(n, (int64_t)tc_wgrad_pick_splits(p.OUT, p.last(), b) * p.OUT * p.last());
    }
    return n;
}

static MlpPlan make_mlp_plan(void* ws, int64_t ws_bytes, const cpb_mlpvae_spec* c, int mode) {
    MlpPlan p;
    memset(&p, 0, sizeof(p));
    const int64_t b = c->base.batch;
    p.B = (int)b; p.IN = kMlpNpix * 3; p.OUT = kMlpNpix * c->base.target_channels; p.z = c->base.z_dim;
    p.zp = z_pad(p.z);
    p.nenc = c->num_encoder; p.ndec = c->num_decoder;
    for (int i = 0; i < p.nenc; ++i) p.enc[i] = c->encoder_sizes[i];
    for (int j = 0; j < p.ndec; ++j) p.dec[j] = c->decoder_sizes[j];
    const int64_t zp = p.zp;
    Arena a(ws, ws_bytes);
    p.x = a.take<float>(b * p.IN);
    for (int i = 0; i < p.nenc; ++i) p.h[i] = a.take<float>(b * p.enc[i]);
    p.heads = a.take<float>(2 * b * zp);
    p.ksplit = a.take<float>((int64_t)kMaxKSplit * 2 * b * zp);
    if (p.zp != p.z) {
        int64_t o = 0;
        auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
        p.pHeads = take(2LL * p.top() * zp); p.pHeadsB = take(2LL * zp); p.pD1 = take(zp * p.dec[0]);
        p.wP = a.take<float>(o);
    }
    if (mode >= CPB_WS_FORWARD) {
        p.y = a.take<float>(b * p.OUT);
        p.zbuf = a.take<float>(b * zp);
        p.kl_rows = a.take<float>(b); p.kl_active = a.take<float>(b); p.frame_loss = a.take<float>(b);
        for (int j = 0; j < p.ndec; ++j) p.g[j] = a.take<float>(b * p.dec[j]);
        p.logits = a.take<float>(b * p.OUT);
    }
    if (mode >= CPB_WS_TRAIN) {
        int64_t widest = 0;
        for (int i = 0; i < p.nenc; ++i) widest = std::max<int64_t>(widest, p.enc[i]);
        for (int j = 0; j < p.ndec; ++j) widest = std::max<int64_t>(widest, p.dec[j]);
        p.ga = a.take<float>(b * widest);
        p.gb = a.take<float>(b * widest);
        p.gz = a.take<float>(b * zp);
        p.gheads = a.take<float>(2 * b * zp);
        int64_t o = 0;
        auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
        for (int i = 1; i < p.nenc; ++i) p.tEnc[i] = take((int64_t)p.enc[i - 1] * p.enc[i]);
        p.tHeads = take(2LL * p.top() * zp);
        for (int j = 0; j < p.ndec; ++j) p.tDec[j] = take((j ? (int64_t)p.dec[j - 1] : zp) * p.dec[j]);
        p.tDec[p.ndec] = take((int64_t)p.last() * p.OUT);
        p.wT = a.take<float>(o);
        // the weight-gradient partials of every layer: consecutive widths of IN, enc..., z_pad, dec..., OUT
        int widths[2 * kMlpMaxLayers + 3], nw = 0;
        widths[nw++] = p.IN;
        for (int i = 0; i < p.nenc; ++i) widths[nw++] = p.enc[i];
        widths[nw++] = p.zp;
        for (int j = 0; j < p.ndec; ++j) widths[nw++] = p.dec[j];
        widths[nw++] = p.OUT;
        int64_t best = 0;
        for (int k = 0; k + 1 < nw; ++k)
            best = std::max<int64_t>(best, (int64_t)wgrad_pick_splits(widths[k], widths[k + 1], b) * widths[k] * widths[k + 1]);
        p.partial = a.take<float>(best);
        p.colsum = a.take<float>(colsum_scratch_floats(b, p.OUT) + colsum_scratch_floats(b, (int)widest));
    }
    // last, so that modes 0 and 1 and every buffer above keep their sizes and offsets
    p.tc = g_math_mode == 2 && mlp_tc_batch_ok(b, p.IN);
    if (p.tc) {
        int64_t o = 0;
        auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
        p.iE1 = take(2LL * p.enc[0] * p.IN);
        if (mode >= CPB_WS_FORWARD) p.iD3f = take(2LL * p.OUT * p.last());
        if (mode >= CPB_WS_TRAIN) p.iD3t = take(2LL * p.last() * p.OUT);
        p.wTc = a.take<float>(o);
        p.tcScratch = a.take<float>(mlp_tc_scratch_floats(p, mode));
    }
    p.bytes = a.off;
    return p;
}

// The weights a call reads besides the parameters: z < z_pad, the zero-padded copies of the z-sized weights (one launch);
// math mode 2, the TF32 weight images (rounded to nearest) of the frame-wide products the call runs (one launch)
static int32_t mlp_relayout_weights(const MlpPlan& pl, const MlpLayout& L, const float* params, bool encoder, bool decoder,
                                    bool backward, cudaStream_t s) {
    RelayoutTable t;
    memset(&t, 0, sizeof(t));
    add_z_padding(t, Latent{pl.B, pl.top(), pl.z, pl.zp, L.off, L.mean()}, true, pl.pHeads, pl.pHeadsB, true, L.off[L.dec(0)],
                  pl.dec[0], pl.pD1);
    CPB_TRY(launch_relayout(params, pl.wP, t, s));
    if (!pl.tc) return CPB_OK;
    TcWeightTable w;
    memset(&w, 0, sizeof(w));
    auto add = [&](int tensor, int64_t dst, int mode, int N, int C) {
        TcWeightJob& j = w.jobs[w.njobs++];
        j.src_off = L.off[tensor]; j.dst_hi = j.dst_lo = dst; j.mode = mode; j.N = N; j.C = C; j.round_nearest = 1;
        j.count = (long long)N * C; w.total += j.count;
    };
    const int out = L.dec(pl.ndec);
    if (encoder) add(L.enc(0), pl.iE1, 3, pl.enc[0], pl.IN);       // [enc0][IN] from the kernel [IN][enc0]
    if (decoder) add(out, pl.iD3f, 3, pl.OUT, pl.last());          // [OUT][dec_last] from the kernel [dec_last][OUT]
    if (backward) add(out, pl.iD3t, 0, pl.last(), pl.OUT);         // the kernel as stored: the data gradient's [N = dec_last][K = OUT]
    ProfScope prof("mlp.tc_weights", s);
    return launch_tc_weights(params, pl.wTc, w, s);
}

// a dense layer: one TF32 pass on the tensor-core tap-GEMM when `image` (its weight image) is given, k-split over
// tcScratch where the reduction is frame-wide; the fp32 SIMT tap-GEMM otherwise
static int32_t mlp_dense(const char* label, const MlpPlan& pl, TapGemmParams p, const float* image, cudaStream_t s) {
    ProfScope prof(label, s);
    if (image == nullptr) return launch_tapgemm(p, s);
    p.wk_hi = p.wk_lo = image;        // single pass: the hi image only (the lo slots of the interleaved image are unused)
    p.passes = 1;
    p.ksplit = tc_tapgemm_pick_ksplit(p.C);
    if (p.ksplit > 1) { p.kpartial = pl.tcScratch; p.kpartial_stride = (long long)p.batch * p.N; }
    return launch_tc_tapgemm(p, s);
}

// math mode 2: out = big[B, I]^T small[B, J] as one TF32 pass on tc_wgrad (I >= 128); transposed: out is [J][I]
static int32_t run_tc_dense_wgrad(const char* label, const float* big, int I, const float* small, int J, int B, float* partial,
                                  float* out, bool transposed, cudaStream_t s) {
    ProfScope prof(label, s);
    WgradParams w;
    memset(&w, 0, sizeof(w));
    w.big = big; w.small = small; w.partial = partial;
    w.batch = B; w.Wb = 1; w.big_pitch = I; w.big_img = I; w.Ho = w.Wo = 1; w.sstride = 1;
    w.ntaps = 1; w.run = I; w.tap_off[0] = 0; w.I = I; w.J = J; w.passes = 1;
    w.splits = tc_wgrad_pick_splits(I, J, B);
    w.m_per_split = align_up(((long long)B + w.splits - 1) / w.splits, 32);
    CPB_TRY(launch_tc_wgrad(w, s));
    if (transposed) return launch_reduce_partials_t(partial, w.splits, I, J, out, s);
    return launch_reduce_partials(partial, w.splits, I, J, I, I, J, out, s);
}

static int32_t mlp_encoder(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_spec* c, const float* params, const void* source,
                           int32_t* flags, cudaStream_t s) {
    const float sscale = c->base.source_dtype == CPB_FRAME_U8 ? 1.f / 255.f : 1.f;
    CPB_TRY(launch_prep_flat(source, c->base.source_dtype, sscale, (long long)pl.B * pl.IN, pl.x, flags, 1, s));
    TapGemmParams p = dense_problem(pl.x, pl.B, pl.IN, params + L.off[L.enc(0)], pl.enc[0], params + L.off[L.enc(0) + 1],
                                    nullptr, pl.h[0], 1);
    CPB_TRY(mlp_dense("mlp.enc.fwd", pl, p, pl.tc ? pl.wTc + pl.iE1 : nullptr, s));
    for (int i = 1; i < pl.nenc; ++i) {
        p = dense_problem(pl.h[i - 1], pl.B, pl.enc[i - 1], params + L.off[L.enc(i)], pl.enc[i], params + L.off[L.enc(i) + 1],
                          nullptr, pl.h[i], 1);
        CPB_TRY(launch_tapgemm(p, s));
    }
    return launch_tapgemm(heads_fwd_problem(Latent{pl.B, pl.top(), pl.z, pl.zp, L.off, L.mean()}, params, pl.h[pl.nenc - 1],
                                            pl.wP + pl.pHeads, pl.wP + pl.pHeadsB, pl.heads), s);
}

static int32_t mlp_decoder(const MlpPlan& pl, const MlpLayout& L, const float* params, const float* zsrc, float* logits, cudaStream_t s) {
    const float* src = zsrc;
    int k = pl.zp;
    for (int j = 0; j < pl.ndec; ++j) {
        const float* w = j == 0 && pl.zp != pl.z ? pl.wP + pl.pD1 : params + L.off[L.dec(j)];
        TapGemmParams p = dense_problem(src, pl.B, k, w, pl.dec[j], params + L.off[L.dec(j) + 1], nullptr, pl.g[j], 1);
        CPB_TRY(launch_tapgemm(p, s));
        src = pl.g[j];
        k = pl.dec[j];
    }
    const int out = L.dec(pl.ndec);
    TapGemmParams p = dense_problem(src, pl.B, k, params + L.off[out], pl.OUT, params + L.off[out + 1], nullptr, logits, 0);
    return mlp_dense("mlp.dec2.fwd", pl, p, pl.tc ? pl.wTc + pl.iD3f : nullptr, s);
}

static int32_t mlp_forward_loss(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_spec* c, const float* params, const void* source,
                                const void* target, const float* eps, bool want_dlogits, int32_t* flags, cudaStream_t s) {
    CPB_TRY(mlp_encoder(pl, L, c, params, source, flags, s));
    CPB_TRY(launch_reparam(pl.heads, eps, pl.B, pl.z, pl.zp, c->base.kl_tolerance, pl.zbuf, pl.kl_rows, pl.kl_active, s));
    CPB_TRY(mlp_decoder(pl, L, params, pl.zbuf, pl.logits, s));
    const float* y = target_is_source(&c->base, source, target) ? pl.x : pl.y;
    if (y == pl.y) {
        const float tscale = c->base.target_dtype == CPB_FRAME_U8 ? c->base.target_u8_scale : 1.f;
        CPB_TRY(launch_prep_flat(target, c->base.target_dtype, tscale, (long long)pl.B * pl.OUT, pl.y, flags, 2, s));
    }
    return launch_recon_loss_flat(pl.logits, y, pl.B, pl.OUT, c->base.loss_type, c->base.loss_scale / (float)pl.B, pl.frame_loss,
                                  want_dlogits ? pl.logits : nullptr, s);
}

static int32_t mlp_backward(const MlpPlan& pl, const MlpLayout& L, const cpb_mlpvae_spec* c, const float* params, const float* eps,
                            float* grads, cudaStream_t s) {
    const int B = pl.B, z = pl.z, zp = pl.zp, ne = pl.nenc, nd = pl.ndec, out = L.dec(nd);
    float* dlog = pl.logits;
    float* cs = pl.colsum;
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    // transposed kernels for the data gradients ([in,out] -> [out,in]); the two head kernels are adjacent (2 "taps").
    // One launch, or one per full table in deep models.
    RelayoutTable t;
    memset(&t, 0, sizeof(t));
    auto add = [&](int tensor, int64_t dst, int taps, int rows, int cols, int rows_pad, int cols_pad) -> int32_t {
        if (t.njobs == kMaxRelayoutJobs) {
            CPB_TRY(launch_relayout(params, pl.wT, t, s));
            memset(&t, 0, sizeof(t));
        }
        add_relayout(t, L.off[tensor], dst, taps, rows, cols, 0, rows_pad, cols_pad);
        return CPB_OK;
    };
    for (int i = 1; i < ne; ++i) CPB_TRY(add(L.enc(i), pl.tEnc[i], 1, pl.enc[i - 1], pl.enc[i], pl.enc[i - 1], pl.enc[i]));
    CPB_TRY(add(L.mean(), pl.tHeads, 2, pl.top(), z, pl.top(), zp));                // [2][z_pad][top]
    CPB_TRY(add(L.dec(0), pl.tDec[0], 1, z, pl.dec[0], zp, pl.dec[0]));              // [dec0][z_pad]
    for (int j = 1; j < nd; ++j) CPB_TRY(add(L.dec(j), pl.tDec[j], 1, pl.dec[j - 1], pl.dec[j], pl.dec[j - 1], pl.dec[j]));
    if (!pl.tc) CPB_TRY(add(out, pl.tDec[nd], 1, pl.last(), pl.OUT, pl.last(), pl.OUT));    // mode 2 reads the TF32 image iD3t instead
    CPB_TRY(launch_relayout(params, pl.wT, t, s));
    TapGemmParams p;
    // ---- output layer.  Mode 2: its weight gradient runs as its transpose dlog^T g_last (I = OUT >= 12 800 rows,
    // J = dec_last columns: tc_wgrad needs I >= 128 and dec_last may be 32), transposed back in the split reduction.
    if (pl.tc)
        CPB_TRY(run_tc_dense_wgrad("mlp.dec2.wgrad", dlog, pl.OUT, pl.g[nd - 1], pl.last(), B, pl.tcScratch, grads + L.off[out], true, s));
    else
        CPB_TRY(run_dense_wgrad("mlp.dec2.wgrad", pl.g[nd - 1], pl.last(), pl.last(), dlog, B, pl.OUT, pl.OUT, pl.partial,
                                grads + L.off[out], s));
    CPB_TRY(launch_colsum(dlog, B, pl.OUT, pl.OUT, grads + L.off[out + 1], cs, s));
    p = dense_problem(dlog, B, pl.OUT, pl.wT + pl.tDec[nd], pl.last(), nullptr, pl.g[nd - 1], pl.ga, 0);   // ga = g(g_last pre-activation)
    CPB_TRY(mlp_dense("mlp.dec2.dgrad", pl, p, pl.tc ? pl.wTc + pl.iD3t : nullptr, s));
    // ---- decoder hidden layers, top down: the gradient alternates between ga and gb; decoder/dense's goes to gz
    float* cur = pl.ga;
    float* other = pl.gb;
    for (int j = nd - 1; j >= 0; --j) {
        const float* in = j ? pl.g[j - 1] : pl.zbuf;
        const int k = j ? pl.dec[j - 1] : zp, k_real = j ? k : z;
        CPB_TRY(run_dense_wgrad("mlp.wgrad", in, k, k_real, cur, B, pl.dec[j], pl.dec[j], pl.partial, grads + L.off[L.dec(j)], s));
        CPB_TRY(launch_colsum(cur, B, pl.dec[j], pl.dec[j], grads + L.off[L.dec(j) + 1], cs, s));
        p = dense_problem(cur, B, pl.dec[j], pl.wT + pl.tDec[j], k, nullptr, j ? pl.g[j - 1] : nullptr, j ? other : pl.gz, 0);
        CPB_TRY(launch_tapgemm(p, s));
        std::swap(cur, other);
    }
    // ---- sampling + KL, heads
    const float* htop = pl.h[ne - 1];
    CPB_TRY(launch_reparam_bwd(pl.heads, eps, pl.gz, pl.kl_active, B, z, zp, c->base.beta * c->base.loss_scale / (float)B, pl.gheads, s));
    // the encoder's gradient alternates between ga and gb so that the first layer's lands in gb at every depth
    cur = ne % 2 == 0 ? pl.ga : pl.gb;
    other = ne % 2 == 0 ? pl.gb : pl.ga;
    CPB_TRY(heads_backward(Latent{B, pl.top(), z, zp, L.off, L.mean()}, "mlp.wgrad", nullptr, htop, pl.gheads, pl.wT + pl.tHeads,
                           cur, pl.partial, cs, grads, s));                                           // cur = g(h_top pre-activation)
    // ---- encoder, top down
    for (int i = ne - 1; i >= 1; --i) {
        CPB_TRY(run_dense_wgrad("mlp.wgrad", pl.h[i - 1], pl.enc[i - 1], pl.enc[i - 1], cur, B, pl.enc[i], pl.enc[i], pl.partial,
                                grads + L.off[L.enc(i)], s));
        CPB_TRY(launch_colsum(cur, B, pl.enc[i], pl.enc[i], grads + L.off[L.enc(i) + 1], cs, s));
        p = dense_problem(cur, B, pl.enc[i], pl.wT + pl.tEnc[i], pl.enc[i - 1], nullptr, pl.h[i - 1], other, 0);
        CPB_TRY(launch_tapgemm(p, s));                                                                  // other = g(h_{i-1} pre-activation)
        std::swap(cur, other);
    }
    if (pl.tc)
        CPB_TRY(run_tc_dense_wgrad("mlp.enc.wgrad", pl.x, pl.IN, cur, pl.enc[0], B, pl.tcScratch, grads + L.off[L.enc(0)], false, s));
    else
        CPB_TRY(run_dense_wgrad("mlp.enc.wgrad", pl.x, pl.IN, pl.IN, cur, B, pl.enc[0], pl.enc[0], pl.partial, grads + L.off[L.enc(0)], s));
    return launch_colsum(cur, B, pl.enc[0], pl.enc[0], grads + L.off[L.enc(0) + 1], cs, s);
}

// every VAE entry point, once its configuration is valid: the device is set up, the workspace given and `need` bytes large
static int32_t check_workspace(const void* workspace, int64_t workspace_bytes, int64_t need) {
    CPB_TRY(ensure_init());
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");
    if (need <= workspace_bytes) return CPB_OK;
    set_error("workspace too small: need %lld bytes, got %lld", (long long)need, (long long)workspace_bytes);
    return CPB_ERR_WORKSPACE_TOO_SMALL;
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

/* debug: byte offsets of the named workspace buffers for (spec's batch, ct, z, frame; mode); returns the count written */
int32_t cpb_debug_vae_spec_buffer_offsets(const cpb_vae_spec* spec, int32_t mode, int64_t* offsets, int32_t capacity) {
    CPB_REQUIRE(spec != nullptr, "cfg is NULL");
    CPB_TRY(check_frame(spec->height, spec->width));
    char* base = (char*)4096;   // fake non-null base: only differences are used
    VaePlan pl = make_plan(base, (int64_t)1 << 60, spec->base.batch, spec->base.target_channels, spec->base.z_dim, mode,
                           make_geo(spec->height, spec->width));
    const float* ptrs[] = {pl.xp, pl.a1, pl.a2, pl.a3, pl.a4, pl.heads, pl.zbuf, pl.d1, pl.b1, pl.b2, pl.b3, pl.logits_p, pl.gA, pl.gB,
                           pl.frame_loss, pl.kl_rows, pl.gz, pl.gheads};
    const int n = (int)(sizeof(ptrs) / sizeof(ptrs[0]));
    // the table only grows at its end: a caller that asks for the first `capacity` entries gets exactly those
    const int written = n < capacity ? n : (capacity > 0 ? capacity : 0);
    for (int i = 0; i < written; ++i) offsets[i] = ptrs[i] ? (int64_t)((const char*)ptrs[i] - base) : -1;
    return written;
}

/* debug: make every later ConvVAE backward pass return right after the named layer group (NULL: run the whole pass) */
int32_t cpb_debug_vae_backward_stop(const char* group) {
    if (group == nullptr) {
        g_backward_stop = nullptr;
        return CPB_OK;
    }
    for (const char* stop : kBackwardStops)
        if (strcmp(group, stop) == 0) {
            g_backward_stop = stop;
            return CPB_OK;
        }
    cpb::set_error("cpb_debug_vae_backward_stop: unknown layer group '%s'", group);
    return CPB_ERR_INVALID_ARGUMENT;
}

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

int32_t cpb_vae_num_tensors(void) { return T_COUNT; }
const char* cpb_vae_tensor_name(int32_t i) { return (i >= 0 && i < T_COUNT) ? kVaeNames[i] : nullptr; }

int32_t cpb_vae_spec_layout(const cpb_vae_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_REQUIRE(spec != nullptr, "spec is NULL");
    const int ct = spec->base.target_channels, z = spec->base.z_dim;
    CPB_REQUIRE(ct == 1 || ct == 3, "target_channels must be 1 or 3, got %d", ct);
    CPB_REQUIRE(z_ok(z), CPB_Z_RULE, z);
    CPB_TRY(check_frame(spec->height, spec->width));
    VaeLayout L = make_layout(ct, z, make_geo(spec->height, spec->width));
    for (int i = 0; i < T_COUNT; ++i) {
        if (offsets) offsets[i] = L.off[i];
        if (sizes) sizes[i] = L.size[i];
        if (shapes) for (int d = 0; d < 4; ++d) shapes[i * 4 + d] = L.shape[i][d];
    }
    if (total) *total = L.total;
    return CPB_OK;
}

int64_t cpb_vae_spec_workspace_bytes(const cpb_vae_spec* spec, int32_t mode) {
    if (spec == nullptr) {
        cpb::set_error("cpb_vae_spec_workspace_bytes: bad arguments: spec is NULL");
        return CPB_ERR_INVALID_ARGUMENT;
    }
    const int batch = spec->base.batch, ct = spec->base.target_channels, z = spec->base.z_dim;
    if (!z_ok(z)) {
        cpb::set_error("cpb_vae_workspace_bytes: bad arguments: " CPB_Z_RULE, z);
        return CPB_ERR_INVALID_ARGUMENT;
    }
    if (!frame_side_ok(spec->height) || !frame_side_ok(spec->width)) {
        cpb::set_error("cpb_vae_workspace_bytes: bad arguments: " CPB_FRAME_RULE, spec->height, spec->width);
        return CPB_ERR_INVALID_ARGUMENT;
    }
    if (batch < 1 || (ct != 1 && ct != 3) || mode < 0 || mode > 2) {
        cpb::set_error("cpb_vae_workspace_bytes: bad arguments");
        return CPB_ERR_INVALID_ARGUMENT;
    }
    return make_plan(nullptr, 0, batch, ct, z, mode, make_geo(spec->height, spec->width)).bytes;
}

// Every ConvVAE compute entry point starts here: the spec is valid and within the batch bound, the device is set up, and
// the plan of `mode` fits the workspace -- all before the first launch
#define CPB_VAE_PLAN(mode)                                                                                                  \
    CPB_TRY(check_spec(spec));                                                                                              \
    const cpb_vae_config* cfg = &spec->base;                                                                                \
    const Geo geo = make_geo(spec->height, spec->width);                                                                    \
    CPB_TRY(check_batch_bound(spec, geo));                                                                                  \
    const VaePlan pl = make_plan(workspace, workspace_bytes, cfg->batch, cfg->target_channels, cfg->z_dim, mode, geo);      \
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));                                                         \
    const VaeLayout L = make_layout(cfg->target_channels, cfg->z_dim, geo);                                                 \
    cudaStream_t s = (cudaStream_t)stream

int32_t cpb_vae_spec_encode(const cpb_vae_spec* spec, const float* params, const void* source, float* mean, float* logvar,
                            int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_VAE_PLAN(CPB_WS_ENCODE);
    CPB_REQUIRE(params && source && mean, "encode: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, false, false, s));
    CPB_TRY(run_encoder(pl, L, cfg, params, source, flags, s));
    return copy_latents_out(pl.heads, pl.zbuf, pl.B, pl.z, pl.zp, mean, logvar, nullptr, s);
}

int32_t cpb_vae_spec_decode(const cpb_vae_spec* spec, const float* params, const float* z, float* reconstruction,
                            void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_VAE_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && z && reconstruction, "decode: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, false, true, false, s));
    if (pl.zp != pl.z) {
        CPB_TRY(launch_pitch_copy(z, pl.z, pl.zbuf, pl.zp, pl.B, s));
        z = pl.zbuf;
    }
    return run_decoder(pl, L, params, z, nullptr, reconstruction, s);
}

int32_t cpb_vae_spec_forward(const cpb_vae_spec* spec, const float* params, const void* source, const void* target,
                             const float* eps, float* losses, float* mean, float* logvar, float* z,
                             float* reconstruction, int32_t* flags, void* workspace, int64_t workspace_bytes,
                             void* stream) {
    CPB_VAE_PLAN(CPB_WS_FORWARD);
    CPB_REQUIRE(params && source && target && losses, "forward: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, true, false, s));
    CPB_TRY(run_forward_loss(pl, L, cfg, params, source, target, eps, false, reconstruction, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, cfg->loss_scale, losses, s));
    return copy_latents_out(pl.heads, pl.zbuf, pl.B, pl.z, pl.zp, mean, logvar, z, s);
}

int32_t cpb_vae_spec_loss_grad(const cpb_vae_spec* spec, const float* params, const void* source, const void* target,
                               const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_VAE_PLAN(CPB_WS_TRAIN);
    CPB_REQUIRE(params && source && target && grads && losses, "loss_grad: NULL pointer");
    CPB_TRY(relayout_weights(pl, L, params, true, true, true, s));
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

int32_t cpb_vae_spec_train_step(const cpb_vae_spec* spec, float* params, float* grads, float* adam_m, float* adam_v,
                                float* adam_powers, float lr, const void* source, const void* target, const float* eps,
                                float* losses, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_TRY(cpb_vae_spec_loss_grad(spec, params, source, target, eps, grads, losses, flags, workspace, workspace_bytes, stream));
    const cpb_vae_config* cfg = &spec->base;
    VaeLayout L = make_layout(cfg->target_channels, cfg->z_dim, make_geo(spec->height, spec->width));
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

// The VAE half of an encode_predict call: the mean of `frames` into latent [B, z]
typedef int32_t (*EncodeMeanFn)(const void* vae, const float* params, const void* frames, float* latent, int32_t* flags,
                                void* workspace, int64_t workspace_bytes, void* stream);

// cpb_encode_predict and cpb_mlpvae_encode_predict: `encode` on the VAE described by `vae` (whose common part is `base`),
// then the state assembly and the PPO forward
static int32_t encode_predict(const cpb_vae_config* base, const void* vae, EncodeMeanFn encode, const float* vae_params,
                              const void* frames, const float* measurements, int32_t num_measurements, const cpb_ppo_config* ppo_cfg,
                              const float* ppo_params, const float* noise, float* latent_tmp, float* state, float* action,
                              float* value, int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes, void* ppo_workspace,
                              int64_t ppo_workspace_bytes, void* stream) {
    CPB_REQUIRE(base && ppo_cfg && frames && latent_tmp && state && action && value, "encode_predict: NULL pointer");
    CPB_REQUIRE(num_measurements >= 0 && (num_measurements == 0 || measurements != nullptr), "encode_predict: bad measurements");
    CPB_REQUIRE(ppo_cfg->state_dim == base->z_dim + num_measurements, "encode_predict: state_dim %d != z_dim %d + %d measurements",
                ppo_cfg->state_dim, base->z_dim, num_measurements);
    const int B = base->batch;
    CPB_TRY(encode(vae, vae_params, frames, latent_tmp, flags, vae_workspace, vae_workspace_bytes, stream));
    const int total = B * ppo_cfg->state_dim;
    assemble_state_kernel<<<cdiv(total, 128), 128, 0, (cudaStream_t)stream>>>(latent_tmp, measurements, B, base->z_dim, num_measurements, state);
    CPB_LAUNCHED();
    return cpb_ppo_forward(ppo_cfg, ppo_params, state, B, noise, action, value, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_vae_spec_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
                                    int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                    float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                                    int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    EncodeMeanFn encode = [](const void* vae, const float* params, const void* frames, float* latent, int32_t* flags, void* ws,
                             int64_t ws_bytes, void* stream) {
        return cpb_vae_spec_encode((const cpb_vae_spec*)vae, params, frames, latent, nullptr, flags, ws, ws_bytes, stream);
    };
    return encode_predict(spec ? &spec->base : nullptr, spec, encode, vae_params, frames, measurements, num_measurements, ppo_cfg,
                          ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace, vae_workspace_bytes,
                          ppo_workspace, ppo_workspace_bytes, stream);
}

static int64_t frame_bytes(const cpb_vae_spec* spec, int dtype, int channels) {
    return (int64_t)spec->height * spec->width * channels * (dtype == CPB_FRAME_U8 ? 1 : 4);
}

int64_t cpb_vae_spec_staging_bytes(const cpb_vae_spec* spec) {
    if (check_spec(spec) != CPB_OK) return CPB_ERR_INVALID_ARGUMENT;
    const cpb_vae_config* cfg = &spec->base;
    const int64_t b = cfg->batch;
    return align_up(b * frame_bytes(spec, cfg->source_dtype, 3), 256) +
           align_up(b * frame_bytes(spec, cfg->target_dtype, cfg->target_channels), 256) +
           align_up(b * cfg->z_dim * 4, 256) + 256;
}

int32_t cpb_vae_spec_train_step_host(const cpb_vae_spec* spec, float* params, float* grads, float* adam_m,
                                     float* adam_v, float* adam_powers, float lr, const void* source_host,
                                     const void* target_host, const float* eps_host, float* losses_host,
                                     int32_t* flags_host, void* staging, int64_t staging_bytes, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_spec(spec));
    CPB_TRY(check_batch_bound(spec, make_geo(spec->height, spec->width)));     // before the uploads
    const cpb_vae_config* cfg = &spec->base;
    CPB_REQUIRE(source_host && target_host && eps_host && losses_host && staging, "train_step_host: NULL pointer");
    CPB_REQUIRE(staging_bytes >= cpb_vae_spec_staging_bytes(spec), "staging buffer too small");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t b = cfg->batch;
    Arena a(staging, staging_bytes);
    const int64_t sb = b * frame_bytes(spec, cfg->source_dtype, 3);
    const int64_t tb = b * frame_bytes(spec, cfg->target_dtype, cfg->target_channels);
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
    CPB_TRY(cpb_vae_spec_train_step(spec, params, grads, adam_m, adam_v, adam_powers, lr, d_src, tgt, d_eps, d_out,
                                    (int32_t*)(d_out + 2), workspace, workspace_bytes, stream));
    float host_out[4];
    CPB_CUDA(cudaMemcpyAsync(host_out, d_out, 16, cudaMemcpyDeviceToHost, s));
    CPB_CUDA(cudaStreamSynchronize(s));
    losses_host[0] = host_out[0];
    losses_host[1] = host_out[1];
    if (flags_host) memcpy(flags_host, &host_out[2], 4);
    return CPB_OK;
}

/* ------------------------------------------------------------------------------- ConvVAE at the default frame */
// The cpb_vae_config entry points: the cpb_vae_spec_* ones at 80x160 (a NULL cfg gives a NULL spec, which they refuse)
struct DefaultFrame {
    cpb_vae_spec spec;
    const cpb_vae_spec* p;
    explicit DefaultFrame(const cpb_vae_config* c) : p(c ? &spec : nullptr) {
        memset(&spec, 0, sizeof(spec));
        if (c) spec.base = *c;
        spec.height = kDefaultH; spec.width = kDefaultW;
    }
    // the layout and workspace queries read target_channels and z_dim (and the batch) only
    DefaultFrame(int32_t batch, int32_t ct, int32_t z) : DefaultFrame(nullptr) {
        spec.base.batch = batch; spec.base.target_channels = ct; spec.base.z_dim = z;
        p = &spec;
    }
};

int32_t cpb_debug_vae_buffer_offsets(int32_t batch, int32_t ct, int32_t z, int32_t mode, int64_t* offsets, int32_t capacity) {
    return cpb_debug_vae_spec_buffer_offsets(DefaultFrame(batch, ct, z).p, mode, offsets, capacity);
}

int32_t cpb_vae_layout(int32_t ct, int32_t z, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    return cpb_vae_spec_layout(DefaultFrame(1, ct, z).p, offsets, sizes, shapes, total);
}

int64_t cpb_vae_workspace_bytes(int32_t batch, int32_t ct, int32_t z, int32_t mode) {
    return cpb_vae_spec_workspace_bytes(DefaultFrame(batch, ct, z).p, mode);
}

int32_t cpb_vae_encode(const cpb_vae_config* cfg, const float* params, const void* source, float* mean,
                       float* logvar, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    return cpb_vae_spec_encode(DefaultFrame(cfg).p, params, source, mean, logvar, flags, workspace, workspace_bytes, stream);
}

int32_t cpb_vae_decode(const cpb_vae_config* cfg, const float* params, const float* z, float* reconstruction,
                       void* workspace, int64_t workspace_bytes, void* stream) {
    return cpb_vae_spec_decode(DefaultFrame(cfg).p, params, z, reconstruction, workspace, workspace_bytes, stream);
}

int32_t cpb_vae_forward(const cpb_vae_config* cfg, const float* params, const void* source, const void* target,
                        const float* eps, float* losses, float* mean, float* logvar, float* z,
                        float* reconstruction, int32_t* flags, void* workspace, int64_t workspace_bytes,
                        void* stream) {
    return cpb_vae_spec_forward(DefaultFrame(cfg).p, params, source, target, eps, losses, mean, logvar, z, reconstruction, flags,
                                workspace, workspace_bytes, stream);
}

int32_t cpb_vae_loss_grad(const cpb_vae_config* cfg, const float* params, const void* source, const void* target,
                          const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    return cpb_vae_spec_loss_grad(DefaultFrame(cfg).p, params, source, target, eps, grads, losses, flags, workspace,
                                  workspace_bytes, stream);
}

int32_t cpb_vae_train_step(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m, float* adam_v,
                           float* adam_powers, float lr, const void* source, const void* target, const float* eps,
                           float* losses, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    return cpb_vae_spec_train_step(DefaultFrame(cfg).p, params, grads, adam_m, adam_v, adam_powers, lr, source, target, eps,
                                   losses, flags, workspace, workspace_bytes, stream);
}

int64_t cpb_vae_staging_bytes(const cpb_vae_config* cfg) { return cpb_vae_spec_staging_bytes(DefaultFrame(cfg).p); }

int32_t cpb_vae_train_step_host(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, float lr, const void* source_host,
                                const void* target_host, const float* eps_host, float* losses_host,
                                int32_t* flags_host, void* staging, int64_t staging_bytes, void* workspace,
                                int64_t workspace_bytes, void* stream) {
    return cpb_vae_spec_train_step_host(DefaultFrame(cfg).p, params, grads, adam_m, adam_v, adam_powers, lr, source_host,
                                        target_host, eps_host, losses_host, flags_host, staging, staging_bytes, workspace,
                                        workspace_bytes, stream);
}

int32_t cpb_encode_predict(const cpb_vae_config* vae_cfg, const float* vae_params, const void* frames, const float* measurements,
                           int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                           float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                           int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    return cpb_vae_spec_encode_predict(DefaultFrame(vae_cfg).p, vae_params, frames, measurements, num_measurements, ppo_cfg,
                                       ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                                       vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

/* ---------------------------------------------------------------------------------------------------- MlpVAE */
int32_t cpb_mlpvae_spec_num_tensors(const cpb_mlpvae_spec* spec) {
    CPB_TRY(check_mlp_spec(spec));
    return 2 * (spec->num_encoder + spec->num_decoder + 3);
}
const char* cpb_mlpvae_spec_tensor_name(const cpb_mlpvae_spec* spec, int32_t i) {
    if (check_mlp_spec(spec) != CPB_OK) return nullptr;
    return mlp_tensor_name(spec->num_encoder, spec->num_decoder, i);
}

int32_t cpb_mlpvae_spec_layout(const cpb_mlpvae_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_TRY(check_mlp_spec(spec));
    MlpLayout L = make_mlp_layout(spec);
    for (int i = 0; i < L.n; ++i) {
        if (offsets) offsets[i] = L.off[i];
        if (sizes) sizes[i] = L.size[i];
        if (shapes) { shapes[i * 4] = L.shape[i][0]; shapes[i * 4 + 1] = L.shape[i][1]; shapes[i * 4 + 2] = 0; shapes[i * 4 + 3] = 0; }
    }
    if (total) *total = L.total;
    return CPB_OK;
}

/* debug: byte offsets of the named MlpVAE workspace buffers for (spec, mode) in the current math mode; returns the count */
int32_t cpb_debug_mlpvae_spec_buffer_offsets(const cpb_mlpvae_spec* spec, int32_t mode, int64_t* offsets, int32_t capacity) {
    CPB_TRY(check_mlp_spec(spec));
    CPB_REQUIRE(mode >= CPB_WS_ENCODE && mode <= CPB_WS_TRAIN, "bad workspace mode %d", mode);
    char* base = (char*)4096;   // fake non-null base: only differences are used
    MlpPlan pl = make_mlp_plan(base, (int64_t)1 << 60, spec, mode);
    const float* ptrs[2 * kMlpMaxLayers + 6];
    int n = 0;
    ptrs[n++] = pl.x;
    for (int i = 0; i < pl.nenc; ++i) ptrs[n++] = pl.h[i];
    ptrs[n++] = pl.heads;
    ptrs[n++] = pl.zbuf;
    for (int j = 0; j < pl.ndec; ++j) ptrs[n++] = pl.g[j];
    ptrs[n++] = pl.logits;
    ptrs[n++] = pl.ga;
    ptrs[n++] = pl.gb;
    for (int i = 0; i < n && i < capacity; ++i) offsets[i] = ptrs[i] ? (int64_t)((const char*)ptrs[i] - base) : -1;
    return n;
}

int64_t cpb_mlpvae_spec_workspace_bytes(const cpb_mlpvae_spec* spec, int32_t mode) {
    if (check_mlp_spec(spec) != CPB_OK || mode < 0 || mode > 2) return CPB_ERR_INVALID_ARGUMENT;
    return make_mlp_plan(nullptr, 0, spec, mode).bytes;
}

int32_t cpb_mlpvae_spec_encode(const cpb_mlpvae_spec* spec, const float* params, const void* source, float* mean, float* logvar,
                               int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_mlp_spec(spec));
    const MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, spec, CPB_WS_ENCODE);
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));
    const MlpLayout L = make_mlp_layout(spec);
    cudaStream_t s = (cudaStream_t)stream;
    CPB_REQUIRE(params && source && mean, "mlp encode: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, true, false, false, s));
    CPB_TRY(mlp_encoder(pl, L, spec, params, source, flags, s));
    return copy_latents_out(pl.heads, pl.zbuf, pl.B, pl.z, pl.zp, mean, logvar, nullptr, s);
}

int32_t cpb_mlpvae_spec_decode(const cpb_mlpvae_spec* spec, const float* params, const float* z, float* reconstruction, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_mlp_spec(spec));
    const MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, spec, CPB_WS_FORWARD);
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));
    const MlpLayout L = make_mlp_layout(spec);
    cudaStream_t s = (cudaStream_t)stream;
    CPB_REQUIRE(params && z && reconstruction, "mlp decode: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, false, true, false, s));
    if (pl.zp != pl.z) {
        CPB_TRY(launch_pitch_copy(z, pl.z, pl.zbuf, pl.zp, pl.B, s));
        z = pl.zbuf;
    }
    CPB_TRY(mlp_decoder(pl, L, params, z, pl.logits, s));
    return launch_sigmoid(pl.logits, reconstruction, (long long)pl.B * pl.OUT, s);
}

int32_t cpb_mlpvae_spec_forward(const cpb_mlpvae_spec* spec, const float* params, const void* source, const void* target, const float* eps,
                                float* losses, float* mean, float* logvar, float* z, float* reconstruction, int32_t* flags,
                                void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_mlp_spec(spec));
    const MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, spec, CPB_WS_FORWARD);
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));
    const MlpLayout L = make_mlp_layout(spec);
    cudaStream_t s = (cudaStream_t)stream;
    CPB_REQUIRE(params && source && target && losses, "mlp forward: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, true, true, false, s));
    CPB_TRY(mlp_forward_loss(pl, L, spec, params, source, target, eps, false, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, spec->base.loss_scale, losses, s));
    CPB_TRY(copy_latents_out(pl.heads, pl.zbuf, pl.B, pl.z, pl.zp, mean, logvar, z, s));
    if (reconstruction) CPB_TRY(launch_sigmoid(pl.logits, reconstruction, (long long)pl.B * pl.OUT, s));
    return CPB_OK;
}

int32_t cpb_mlpvae_spec_loss_grad(const cpb_mlpvae_spec* spec, const float* params, const void* source, const void* target,
                                  const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
    CPB_TRY(check_mlp_spec(spec));
    const MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, spec, CPB_WS_TRAIN);
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));
    const MlpLayout L = make_mlp_layout(spec);
    cudaStream_t s = (cudaStream_t)stream;
    CPB_REQUIRE(params && source && target && grads && losses, "mlp loss_grad: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, true, true, true, s));
    CPB_TRY(mlp_forward_loss(pl, L, spec, params, source, target, eps, true, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, spec->base.loss_scale, losses, s));
    return mlp_backward(pl, L, spec, params, eps, grads, s);
}

int32_t cpb_mlpvae_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
                                  int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                  float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                                  int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    EncodeMeanFn encode = [](const void* vae, const float* params, const void* frames, float* latent, int32_t* flags, void* ws,
                             int64_t ws_bytes, void* stream) {
        return cpb_mlpvae_spec_encode((const cpb_mlpvae_spec*)vae, params, frames, latent, nullptr, flags, ws, ws_bytes, stream);
    };
    return encode_predict(spec ? &spec->base : nullptr, spec, encode, vae_params, frames, measurements, num_measurements, ppo_cfg,
                          ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace, vae_workspace_bytes,
                          ppo_workspace, ppo_workspace_bytes, stream);
}

/* The two-per-side entry points: the spec entry points on {enc1, enc2} / {dec1, dec2} */
static int32_t spec_of(const cpb_mlpvae_config* c, cpb_mlpvae_spec* spec) {
    CPB_REQUIRE(c != nullptr, "mlp cfg is NULL");
    memset(spec, 0, sizeof(*spec));
    spec->base = c->base;
    spec->num_encoder = 2; spec->encoder_sizes[0] = c->enc1; spec->encoder_sizes[1] = c->enc2;
    spec->num_decoder = 2; spec->decoder_sizes[0] = c->dec1; spec->decoder_sizes[1] = c->dec2;
    return CPB_OK;
}
#define CPB_MLP_SPEC_OF(cfg)   \
    cpb_mlpvae_spec spec;      \
    CPB_TRY(spec_of(cfg, &spec));

int32_t cpb_mlpvae_num_tensors(void) { return 2 * (2 + 2 + 3); }
const char* cpb_mlpvae_tensor_name(int32_t i) { return mlp_tensor_name(2, 2, i); }

int32_t cpb_mlpvae_layout(const cpb_mlpvae_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_mlpvae_spec_layout(&spec, offsets, sizes, shapes, total);
}

int32_t cpb_debug_mlpvae_buffer_offsets(const cpb_mlpvae_config* cfg, int32_t mode, int64_t* offsets, int32_t capacity) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_debug_mlpvae_spec_buffer_offsets(&spec, mode, offsets, capacity);
}

int64_t cpb_mlpvae_workspace_bytes(const cpb_mlpvae_config* cfg, int32_t mode) {
    cpb_mlpvae_spec spec;
    if (spec_of(cfg, &spec) != CPB_OK) return CPB_ERR_INVALID_ARGUMENT;
    return cpb_mlpvae_spec_workspace_bytes(&spec, mode);
}

int32_t cpb_mlpvae_encode(const cpb_mlpvae_config* cfg, const float* params, const void* source, float* mean, float* logvar,
                          int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_mlpvae_spec_encode(&spec, params, source, mean, logvar, flags, workspace, workspace_bytes, stream);
}

int32_t cpb_mlpvae_decode(const cpb_mlpvae_config* cfg, const float* params, const float* z, float* reconstruction, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_mlpvae_spec_decode(&spec, params, z, reconstruction, workspace, workspace_bytes, stream);
}

int32_t cpb_mlpvae_forward(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target, const float* eps,
                           float* losses, float* mean, float* logvar, float* z, float* reconstruction, int32_t* flags,
                           void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_mlpvae_spec_forward(&spec, params, source, target, eps, losses, mean, logvar, z, reconstruction, flags, workspace,
                                   workspace_bytes, stream);
}

int32_t cpb_mlpvae_loss_grad(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target, const float* eps,
                             float* grads, float* losses, int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_SPEC_OF(cfg);
    return cpb_mlpvae_spec_loss_grad(&spec, params, source, target, eps, grads, losses, flags, workspace, workspace_bytes, stream);
}

}  // extern "C"
