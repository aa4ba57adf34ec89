// The MlpVAE behind the C ABI (reference vae/models.py:271-299, build_mlp): flatten -> one dense relu layer per encoder
// size -> [mean | logstd_sq] -> sample -> one dense relu layer per decoder size -> the output layer, dense 12800*Ct ->
// logits.  Same loss / sampling / Adam kernels as the ConvVAE; the layers run on the fp32 SIMT tap-GEMM (dense form) and
// the SIMT weight-gradient kernel, except in math mode 2: there the five frame-wide products -- the first encoder layer's
// forward and weight gradient, the output layer's forward, data gradient and weight gradient -- run as ONE TF32 wgmma pass
// with both operands rounded to nearest (the forward passes and the data gradient on the tensor-core tap-GEMM, k-split
// where they reduce over a frame, the weight gradients on tc_wgrad).  Profile labels call the output layer "dec2" at every
// depth (its name in the default two-per-side model).  Every cpb_mlpvae_* entry point but the encode_predict ones
// (actor.cu) is here.
#include <algorithm>

#include "vae_shared.cuh"

namespace cpb {

// The MlpVAE keeps the reference's 80x160 input (its own frame size is a separate spec)
constexpr int kMlpNpix = kDefaultH * kDefaultW;
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
        j.ksplit = tc_tapgemm_pick_ksplit(C) > 1;     // the split mlp_dense picks for this layer (one tap: K = C)
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

}  // namespace cpb

using namespace cpb;

extern "C" {

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

// Every MlpVAE compute entry point starts here: the spec is valid, the device is set up, and the plan of `mode` fits the
// workspace -- all before the first launch
#define CPB_MLP_PLAN(mode)                                                                                                  \
    CPB_TRY(check_mlp_spec(spec));                                                                                          \
    const MlpPlan pl = make_mlp_plan(workspace, workspace_bytes, spec, mode);                                               \
    CPB_TRY(check_workspace(workspace, workspace_bytes, pl.bytes));                                                         \
    const MlpLayout L = make_mlp_layout(spec);                                                                              \
    cudaStream_t s = (cudaStream_t)stream

int32_t cpb_mlpvae_spec_encode(const cpb_mlpvae_spec* spec, const float* params, const void* source, float* mean, float* logvar,
                               int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_ENCODE);
    CPB_REQUIRE(params && source && mean, "mlp encode: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, true, false, false, s));
    CPB_TRY(mlp_encoder(pl, L, spec, params, source, flags, s));
    return copy_latents_out(pl.heads, pl.zbuf, pl.B, pl.z, pl.zp, mean, logvar, nullptr, s);
}

int32_t cpb_mlpvae_spec_decode(const cpb_mlpvae_spec* spec, const float* params, const float* z, float* reconstruction, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_MLP_PLAN(CPB_WS_FORWARD);
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
    CPB_MLP_PLAN(CPB_WS_FORWARD);
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
    CPB_MLP_PLAN(CPB_WS_TRAIN);
    CPB_REQUIRE(params && source && target && grads && losses, "mlp loss_grad: NULL pointer");
    CPB_TRY(mlp_relayout_weights(pl, L, params, true, true, true, s));
    CPB_TRY(mlp_forward_loss(pl, L, spec, params, source, target, eps, true, flags, s));
    CPB_TRY(launch_finalize_losses(pl.frame_loss, pl.kl_rows, pl.B, spec->base.loss_scale, losses, s));
    return mlp_backward(pl, L, spec, params, eps, grads, s);
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
