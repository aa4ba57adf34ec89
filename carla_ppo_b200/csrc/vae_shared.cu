// The code both VAEs run (see vae_shared.cuh): the configuration and workspace checks, the dense tap-GEMM problem and its
// weight gradient, the weight re-layout jobs, and the latent block -- the two heads, the z_pad padding and the latent copy-out.
#include "vae_shared.cuh"

namespace cpb {

int z_pad(int z) { return (int)align_up(z, 64); }

bool z_ok(int z) { return z >= 4 && z % 4 == 0 && z <= 1024; }

int32_t check_cfg(const cpb_vae_config* cfg) {
    CPB_REQUIRE(cfg != nullptr, "cfg is NULL");
    CPB_REQUIRE(cfg->batch >= 1 && cfg->batch <= (1 << 20), "batch=%d out of range", cfg->batch);
    CPB_REQUIRE(cfg->target_channels == 1 || cfg->target_channels == 3, "target_channels must be 1 or 3, got %d", cfg->target_channels);
    CPB_REQUIRE(z_ok(cfg->z_dim), CPB_Z_RULE, cfg->z_dim);
    CPB_REQUIRE(cfg->loss_type >= 0 && cfg->loss_type <= 2, "unknown loss_type %d", cfg->loss_type);
    CPB_REQUIRE(cfg->source_dtype == CPB_FRAME_F32 || cfg->source_dtype == CPB_FRAME_U8, "bad source_dtype");
    CPB_REQUIRE(cfg->target_dtype == CPB_FRAME_F32 || cfg->target_dtype == CPB_FRAME_U8, "bad target_dtype");
    return CPB_OK;
}

int32_t check_workspace(const void* workspace, int64_t workspace_bytes, int64_t need) {
    CPB_TRY(ensure_init());
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");
    if (need <= workspace_bytes) return CPB_OK;
    set_error("workspace too small: need %lld bytes, got %lld", (long long)need, (long long)workspace_bytes);
    return CPB_ERR_WORKSPACE_TOO_SMALL;
}

TapGemmParams base_params() {
    TapGemmParams p;
    memset(&p, 0, sizeof(p));
    p.nclass = 1;
    p.ybatch = 1;
    p.ksplit = 1;
    return p;
}

TapGemmParams dense_problem(const float* src, int B, int K, const float* W, int N, const float* bias,
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

int32_t run_dense_wgrad(const char* label, const float* x, int K, int k_real, const float* g, int B, int J, int j_real,
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

void add_relayout(RelayoutTable& t, int64_t src, int64_t dst, int taps, int rows, int cols, int mode,
                  int rows_pad, int cols_pad) {
    RelayoutJob& j = t.jobs[t.njobs++];
    j.src_off = src; j.dst_off = dst; j.taps = taps; j.rows = rows; j.cols = cols; j.mode = mode;
    j.rows_pad = rows_pad; j.cols_pad = cols_pad;
    j.count = (long long)taps * rows_pad * cols_pad;
    t.total += j.count;
}

TapGemmParams heads_fwd_problem(const Latent& h, const float* params, const float* x, const float* wp, const float* bp,
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

int32_t heads_backward(const Latent& h, const char* wgrad_label, const char* dgrad_label, const float* x, const float* gheads,
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

void add_z_padding(RelayoutTable& t, const Latent& h, bool heads, int64_t wp, int64_t bp, bool dec, int64_t dec_off,
                   int N, int64_t dp) {
    if (h.zp == h.z) return;
    if (heads) {
        add_relayout(t, h.off[h.mean], wp, 2, h.K, h.z, 1, h.K, h.zp);
        add_relayout(t, h.off[h.mean + 1], bp, 1, 1, h.z, 1, 1, h.zp);
        add_relayout(t, h.off[h.mean + 3], bp + h.zp, 1, 1, h.z, 1, 1, h.zp);
    }
    if (dec) add_relayout(t, dec_off, dp, 1, h.z, N, 1, h.zp, N);
}

bool target_is_source(const cpb_vae_config* c, const void* source, const void* target) {
    return target == source && c->target_channels == 3 && c->target_dtype == c->source_dtype &&
           (c->target_dtype == CPB_FRAME_F32 || c->target_u8_scale == 1.f / 255.f);
}

int32_t copy_latents_out(const float* heads, const float* zbuf, int B, int z, int zp, float* mean, float* logvar,
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

}  // namespace cpb
