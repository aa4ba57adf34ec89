// The ConvVAE behind the C ABI (include/carla_ppo_b200.h): geometry, parameter layout, workspace plan, layer table and
// passes, and every cpb_vae_* entry point with its 80x160 twin.
// Replaces the TF graph built by reference vae/models.py:85-142 + 249-266 and the sess.run calls of
// VAE.encode / generate_from_latent / reconstruct / evaluate / train_one_epoch (:188-231).
#include <algorithm>

#include "vae_shared.cuh"

namespace cpb {

// ---------------------------------------------------------------------------------------------
// geometry (layer table SURVEY appendix A.1).  The source frame is H x W x 3 (80x160 by default, reference
// vae_common.py:18-20); the encoder's four 4x4 stride-2 VALID convolutions give H1 = H/2 - 1, H2 = H/4 - 2, H3 = H/8 - 2,
// H4 = H/16 - 2 (the same in W), and the decoder (dense1 -> [H4, W4, 256] -> deconvolutions with kernels 4, 4, 5, 4)
// maps H4 back to exactly H only when H is a multiple of 16 (reference vae/models.py:265 asserts it).
// ---------------------------------------------------------------------------------------------
struct Side { int H, W, C; };
constexpr int C1 = 32, C4 = 256;
constexpr int kSideChannels[5] = {3, C1, 64, 128, C4};
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

// ---------------------------------------------------------------------------------------------
// passes
// ---------------------------------------------------------------------------------------------
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

}  // namespace cpb

using namespace cpb;

extern "C" {

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
    const bool spec_ok = check_spec(spec) == CPB_OK;
    if (spec_ok && mode >= 0 && mode <= 2)
        return make_plan(nullptr, 0, spec->base.batch, spec->base.target_channels, spec->base.z_dim, mode,
                         make_geo(spec->height, spec->width)).bytes;
    char why[512];     // check_spec's reason, copied out of the error buffer that set_error overwrites
    if (spec_ok) snprintf(why, sizeof(why), "workspace mode %d is not 0, 1 or 2", mode);
    else snprintf(why, sizeof(why), "%s", cpb_last_error());
    cpb::set_error("cpb_vae_spec_workspace_bytes: bad arguments: %s", why);
    return CPB_ERR_INVALID_ARGUMENT;
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
// The cpb_vae_config entry points: the cpb_vae_spec_* ones at 80x160 (DefaultFrame)
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

}  // extern "C"
