// The device code both PPO learn paths run: the launch-per-kernel kernels (ppo.cu) and the persistent learn() kernel
// (ppo_persistent.cu).  The small tile GEMM and its job builders, the per-sample Gaussian and categorical heads, the loss
// finalisation and the gradient-norm pieces.  Everything here is file-local to each includer (an anonymous namespace),
// like the kernels that inline it.
#pragma once
#include "ppo.cuh"

namespace cpb {
namespace {

// ---------------------------------------------------------------------------------------------
// small tile GEMM: C[M,N] (+)= A'[M,K] * B'[K,N], 32x32 tile, 128 threads, 2x4 per thread
// ---------------------------------------------------------------------------------------------
constexpr int TS = 32;   // tile edge
constexpr int TK = 64;   // reduction chunk (one global round trip per chunk: keep the chunk count low)

// operand access descriptors (element (o, r) = output index o, reduction index r)
struct Operand {
    const float* p;
    long long so, sr;       // strides for the output / reduction index
    const int32_t* gather;  // optional row gather applied to whichever index has the larger stride
    int gather_on_o;        // 1: gather indexes o, 0: gather indexes r
};

// GATHER: 0 = none, 1 = the A operand's output index goes through `gather`, 2 = its reduction index does.
// Compile-time so that the 16 loads of a chunk stay independent (a run-time check serialised them: each
// value load waited on a predicated index load that reused the same register).
template <int GATHER>
__device__ __forceinline__ long long a_offset(const Operand& a, int o, int r) {
    if (GATHER == 1) return (long long)__ldg(a.gather + o) * a.so + (long long)r * a.sr;      // the index vectors are launch inputs
    if (GATHER == 2) return (long long)o * a.so + (long long)__ldg(a.gather + r) * a.sr;
    return (long long)o * a.so + (long long)r * a.sr;
}

struct GemmJob {
    Operand a, b;            // a: (m, r), b: (n, r)
    int M, N, R;
    float* c;                // [M, ldc]
    int ldc;
    const float* bias;       // [N] or null
    const float* mask;       // [M, ldc] or null: out *= mask > 0
    int relu;
    float* colsum;           // [N] or null: colsum[n] = sum_r b(n, r)   (bias gradient; blockIdx.x == 0 only)
};

struct GemmBatch {
    GemmJob job[6];       // independent GEMMs of one launch (blockIdx.z); all with the same gather mode
};

// One 32x32 output tile of job J by a GROUP of kTileThreads = 128 threads (tid = 0..127), 2x4 outputs per thread.  `sync()` is
// the group's barrier: __syncthreads in the stand-alone kernel (one group per CTA), a named barrier in the persistent learn()
// kernel (two groups per CTA).  As / Bs: the group's double-buffered operand tiles [2][TK][TS + 4].
// (Round 1 used 64 threads with 4x4 outputs: 1024 dependent-issue FMAs per thread and 64-wide chunk made every K = 500 tile
// a ~12 us chain; with 128 threads the per-chunk FMA chain halves and twice the warps hide the chunk's global round trip.)
constexpr int kTileThreads = 128;

template <int GATHER, typename Sync>
__device__ __forceinline__ void gemm_tile(const GemmJob& J, int m0, int n0, bool first_m_tile, int tid,
                                          float (*As)[TK][TS + 4], float (*Bs)[TK][TS + 4], Sync sync) {
    const int tx = tid & 7, ty = tid >> 3;      // 8 x 16 threads, 2 rows x 4 columns each
    float acc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float csum = 0.f;                            // column-sum lane (threads 0..31 own column n0+tid)
    const bool do_colsum = J.colsum != nullptr && first_m_tile;
    const bool a_ofast = J.a.so <= J.a.sr, b_ofast = J.b.so <= J.b.sr;

    constexpr int EPT = TS * TK / kTileThreads;  // elements per thread per operand and chunk
    float ra[EPT], rb[EPT];
    auto fetch_chunk = [&](int r0) {
        // TS*TK elements per operand; the faster-varying thread index follows the contiguous memory direction
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int f = tid + e * kTileThreads;
            int o, r;
            if (a_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            ra[e] = (m0 + o < J.M && r0 + r < J.R) ? __ldcg(J.a.p + a_offset<GATHER>(J.a, m0 + o, r0 + r)) : 0.f;
            if (b_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            rb[e] = (n0 + o < J.N && r0 + r < J.R) ? __ldcg(J.b.p + (long long)(n0 + o) * J.b.so + (long long)(r0 + r) * J.b.sr) : 0.f;
        }
    };
    fetch_chunk(0);
    int buf = 0;
    for (int r0 = 0; r0 < J.R; r0 += TK, buf ^= 1) {
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int f = tid + e * kTileThreads;
            int o, r;
            if (a_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            As[buf][r][o] = ra[e];
            if (b_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            Bs[buf][r][o] = rb[e];
        }
        sync();
        if (r0 + TK < J.R) fetch_chunk(r0 + TK);
#pragma unroll
        for (int k = 0; k < TK; ++k) {
            const float2 a = *reinterpret_cast<const float2*>(&As[buf][k][ty * 2]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float av[2] = {a.x, a.y};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (do_colsum && tid < 32) {
#pragma unroll
            for (int k = 0; k < TK; ++k) csum += Bs[buf][k][tid];
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int m = m0 + ty * 2 + i;
        if (m >= J.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= J.N) continue;
            float v = acc[i][j] + (J.bias ? __ldcg(J.bias + n) : 0.f);
            if (J.relu) v = fmaxf(v, 0.f);
            if (J.mask) v = __ldcg(J.mask + (long long)m * J.ldc + n) > 0.f ? v : 0.f;
            J.c[(long long)m * J.ldc + n] = v;
        }
    }
    if (do_colsum && tid < 32 && n0 + tid < J.N) J.colsum[n0 + tid] = csum;
    sync();          // the next tile of this group reuses As / Bs
}

// Y[B,N] = act(X[B,K] W[K,N] + b)
__host__ __device__ GemmJob fwd_job(const float* x, const int32_t* idx, int B, int K, const float* w, int N, const float* bias,
                float* y, int relu) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{x, K, 1, idx, 1};
    j.b = Operand{w, 1, N, nullptr, 0};
    j.M = B; j.N = N; j.R = K; j.c = y; j.ldc = N; j.bias = bias; j.relu = relu;
    return j;
}
// dX[B,K] = (dY[B,N] W[K,N]^T) * (H > 0)
__host__ __device__ GemmJob bwd_data_job(const float* dy, int B, int N, const float* w, int K, const float* h, float* dx) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{dy, N, 1, nullptr, 0};
    j.b = Operand{w, N, 1, nullptr, 0};       // b(k, n) = W[k*N + n]
    j.M = B; j.N = K; j.R = N; j.c = dx; j.ldc = K; j.mask = h;
    return j;
}
// gW[K,N] = X[B,K]^T dY[B,N];  gb[N] = colsum(dY)
__host__ __device__ GemmJob bwd_weight_job(const float* x, const int32_t* idx, int B, int K, const float* dy, int N, float* gw, float* gb) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{x, 1, K, idx, 0};           // a(k, b) = X[b*K + k]
    j.b = Operand{dy, 1, N, nullptr, 0};      // b(n, b) = dY[b*N + n]
    j.M = K; j.N = N; j.R = B; j.c = gw; j.ldc = N; j.colsum = gb;
    return j;
}

// Forward jobs of layer l: one per trunk that has it (layer 0 reads the states through idx)
__host__ __device__ __forceinline__ int trunk_fwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       const float* params, const float* states, const int32_t* idx, int B,
                                                       int l, GemmJob* jobs) {
    int n = 0;
    for (int t = 0; t < 2; ++t) {
        if (l >= trunk_depth(sp, t)) continue;
        const float* in = l ? trunk_buf(pl.h, sp, t, l - 1, B) : states;
        jobs[n++] = fwd_job(in, l ? nullptr : idx, B, trunk_in(sp, t, l), params + L.off[L.w(t, l)], trunk_width(sp, t, l),
                            params + L.off[L.b(t, l)], trunk_buf(pl.h, sp, t, l, B), 1);
    }
    return n;
}

// Backward jobs of layer l: per trunk that has it, the weight and bias gradients and (l > 0) the masked data gradient into
// layer l - 1.  Layer 0 reads the states through idx, so its jobs gather (GATHER 2 when idx != null) and the rest do not.
__host__ __device__ __forceinline__ int trunk_bwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       const float* params, float* grads, const float* states,
                                                       const int32_t* idx, int B, int l, GemmJob* jobs) {
    int n = 0;
    for (int t = 0; t < 2; ++t) {
        if (l >= trunk_depth(sp, t)) continue;
        const float* in = l ? trunk_buf(pl.h, sp, t, l - 1, B) : states;
        jobs[n++] = bwd_weight_job(in, l ? nullptr : idx, B, trunk_in(sp, t, l), trunk_buf(pl.dh, sp, t, l, B),
                                   trunk_width(sp, t, l), grads + L.off[L.w(t, l)], grads + L.off[L.b(t, l)]);
    }
    if (l > 0)
        for (int t = 0; t < 2; ++t) {
            if (l >= trunk_depth(sp, t)) continue;
            jobs[n++] = bwd_data_job(trunk_buf(pl.dh, sp, t, l, B), B, trunk_width(sp, t, l), params + L.off[L.w(t, l)],
                                     trunk_in(sp, t, l), trunk_buf(pl.h, sp, t, l - 1, B), trunk_buf(pl.dh, sp, t, l - 1, B));
        }
    return n;
}

// Weight and bias gradients of the action and value heads: gWm[Hp,N] = hp^T dpre, gbm = colsum(dpre); gWv[Hv,1] = hv^T dv
// (N: the head's columns, num_actions for the Gaussian head, the logits for the categorical one)
__host__ __device__ __forceinline__ void head_bwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       float* grads, int B, int N, GemmJob* jobs) {
    jobs[0] = bwd_weight_job(trunk_buf(pl.h, sp, 0, sp.num_policy - 1, B), nullptr, B, trunk_last(sp, 0), pl.dpre,
                             N, grads + L.off[L.wm()], grads + L.off[L.bm()]);
    jobs[1] = bwd_weight_job(trunk_buf(pl.h, sp, 1, sp.num_value - 1, B), nullptr, B, trunk_last(sp, 1), pl.dv, 1,
                             grads + L.off[L.wv()], grads + L.off[L.bv()]);
}

// ---------------------------------------------------------------------------------------------
// per-sample head: action mean, value, log-prob, ratio, losses and the gradients w.r.t. the two
// trunk outputs (Hp and Hv wide).  One warp per sample.
// ---------------------------------------------------------------------------------------------
constexpr float kLogSqrt2Pi = 0.9189385175704956f;
constexpr float kEntropyConst = 1.4189385175704956f;

struct HeadArgs {
    const float* hp;       // [B,Hp] policy trunk output (post-relu)
    const float* hv;       // [B,Hv] value trunk output (post-relu), may be null (old policy)
    const float* wm; const float* bm; const float* logstd;   // action head
    const float* wv; const float* bv;                        // value head
    const float* actions; const float* returns; const float* adv;   // [T,A], [T], [T] (gathered through idx)
    const int32_t* idx;
    const float* logp_old_in;   // [T] gathered through idx (learn path) or [B] ungathered (train_step path)
    int logp_old_gathered;
    int B, Hp, Hv, A;
    float low[kMaxActions], high[kMaxActions];
    float eps_clip, value_scale, entropy_scale;
    // outputs
    float* logp_out;       // [B] (old-policy pass: log-prob only)
    float* mu_out;         // [B,A] or null
    float* v_out;          // [B] or null
    float* dpre;           // [B,A] gradient w.r.t. the action head pre-activation
    float* dv;             // [B]   gradient w.r.t. the value output
    float* dhp;            // [B,Hp] masked gradient w.r.t. policy trunk output
    float* dhv;            // [B,Hv] masked gradient w.r.t. value trunk output
    float* partial;        // [nblocks][8]: policy, value, ratio sums, logstd grads (3..3+A), approx-KL sum (7)
    const float* noise;    // predict path: [B,A] or null
    float* action_out;     // predict path
    int kl_term;           // training head: add (r - 1) - log r to slot 7 (options entry points only)
    // categorical head only (A = K components): N logits, component k at [coff[k], coff[k+1]); dpre / mu_out are [B,N]
    int N;
    int coff[kMaxActions + 1];
};

// The head arguments every pass shares (weights, shapes, the spec's constants); each caller sets its pass's inputs and outputs
__host__ __device__ __forceinline__ HeadArgs head_args(const cpb_ppo_spec& sp, const HeadShape& hs, const PpoLayout& L,
                                                       const float* params, int B) {
    const cpb_ppo_config& c = sp.base;
    HeadArgs h{};
    h.wm = params + L.off[L.wm()]; h.bm = params + L.off[L.bm()]; h.logstd = params + L.off[L.logstd()];
    h.wv = params + L.off[L.wv()]; h.bv = params + L.off[L.bv()];
    h.B = B; h.Hp = trunk_last(sp, 0); h.Hv = trunk_last(sp, 1); h.A = c.num_actions;
    for (int k = 0; k < kMaxActions; ++k) { h.low[k] = c.action_low[k]; h.high[k] = c.action_high[k]; }
    h.eps_clip = c.epsilon; h.value_scale = c.value_scale; h.entropy_scale = c.entropy_scale;
    h.N = hs.N;
    for (int k = 0; k < 5; ++k) h.coff[k] = hs.off[k];
    return h;
}

// mode 0: log-prob only (old policy); mode 1: full training head; mode 2: predict (mu / sampled action, value)
// one sample (row b) by one warp; MODE 1 adds its loss terms to vals[8]
template <int MODE>
__device__ __forceinline__ void gauss_head_row(const HeadArgs& a, int b, int lane, float* vals) {
    {
        const float* h = a.hp + (long long)b * a.Hp;
        const float* g = MODE != 0 ? a.hv + (long long)b * a.Hv : nullptr;
        float pre[kMaxActions] = {0.f, 0.f, 0.f, 0.f};
        float vsum = 0.f;
        // one loop over both trunk outputs: with Hp == Hv every lane sums in the order of a fused loop
        const int hmax = MODE != 0 && a.Hv > a.Hp ? a.Hv : a.Hp;
        for (int j = lane; j < hmax; j += 32) {
            if (j < a.Hp) {
                const float hv = h[j];
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k)
                    if (k < a.A) pre[k] = fmaf(hv, a.wm[j * a.A + k], pre[k]);
            }
            if (MODE != 0 && j < a.Hv) vsum = fmaf(g[j], a.wv[j], vsum);
        }
#pragma unroll
        for (int k = 0; k < kMaxActions; ++k) pre[k] = warp_sum(pre[k]);
        if (MODE != 0) vsum = warp_sum(vsum);
        const int row = a.idx != nullptr ? a.idx[b] : b;
        float t[kMaxActions], mu[kMaxActions], diff[kMaxActions], sigma[kMaxActions];
        float logp = 0.f;
#pragma unroll
        for (int k = 0; k < kMaxActions; ++k) {
            if (k >= a.A) continue;
            t[k] = tanhf(pre[k] + a.bm[k]);
            mu[k] = a.low[k] + ((t[k] + 1.f) * 0.5f) * (a.high[k] - a.low[k]);
            sigma[k] = expf(a.logstd[k]);
            if (MODE != 2) {
                diff[k] = (a.actions[(long long)row * a.A + k] - mu[k]) / sigma[k];
                logp += -0.5f * diff[k] * diff[k] - (kLogSqrt2Pi + a.logstd[k]);
            }
        }
        if (MODE == 0) {
            if (lane == 0) a.logp_out[b] = logp;
        } else if (MODE == 2) {
            const float v = vsum + a.bv[0];
            if (lane == 0) {
                a.v_out[b] = v;
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k) {
                    if (k >= a.A) continue;
                    float act = mu[k];
                    if (a.noise != nullptr) act = fminf(fmaxf(fmaf(a.noise[(long long)b * a.A + k], sigma[k], mu[k]), a.low[k]), a.high[k]);
                    a.action_out[(long long)b * a.A + k] = act;
                }
            }
        } else {
            const float v = vsum + a.bv[0];
            const float logp_old = a.logp_old_in[a.logp_old_gathered ? row : b];
            const float ratio = expf(logp - logp_old);
            const float adv = a.adv[row], ret = a.returns[row];
            const float unclipped = ratio * adv;
            const float clipped = fminf(fmaxf(ratio, 1.f - a.eps_clip), 1.f + a.eps_clip) * adv;
            const float inv_b = 1.f / (float)a.B;
            // d(-mean(min(u, c)))/d ratio: tf.minimum routes to u when u <= c; the clipped branch has
            // zero slope outside the clip range (inside it u == c and the first branch is taken).
            const float dratio = unclipped <= clipped ? -adv * inv_b : 0.f;
            const float dlogp = dratio * ratio;
            const float dvv = a.value_scale * 2.f * inv_b * (v - ret);
            float dp[kMaxActions] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < kMaxActions; ++k) {
                if (k >= a.A) continue;
                const float dmu = dlogp * diff[k] / sigma[k];
                dp[k] = dmu * 0.5f * (a.high[k] - a.low[k]) * (1.f - t[k] * t[k]);
            }
            if (lane == 0) {
                a.dv[b] = dvv;
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k)
                    if (k < a.A) a.dpre[(long long)b * a.A + k] = dp[k];
                if (a.mu_out != nullptr)
#pragma unroll
                    for (int k = 0; k < kMaxActions; ++k)
                        if (k < a.A) a.mu_out[(long long)b * a.A + k] = mu[k];
                if (a.v_out != nullptr) a.v_out[b] = v;
            }
            for (int j = lane; j < hmax; j += 32) {
                if (j < a.Hp) {
                    float s = 0.f;
#pragma unroll
                    for (int k = 0; k < kMaxActions; ++k)
                        if (k < a.A) s = fmaf(dp[k], a.wm[j * a.A + k], s);
                    a.dhp[(long long)b * a.Hp + j] = h[j] > 0.f ? s : 0.f;
                }
                if (j < a.Hv) a.dhv[(long long)b * a.Hv + j] = g[j] > 0.f ? dvv * a.wv[j] : 0.f;
            }
            vals[0] += fminf(unclipped, clipped);
            vals[1] += (v - ret) * (v - ret);
            vals[2] += ratio;
#pragma unroll
            for (int k = 0; k < kMaxActions; ++k)
                if (k < a.A) vals[3 + k] += dlogp * (diff[k] * diff[k] - 1.f);
            if (a.kl_term) vals[7] += (ratio - 1.f) - (logp - logp_old);   // approximate KL (Stable-Baselines3's estimator)
        }
    }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// logit i (< 64) of a row whose lane l holds logits l in v0 and l + 32 in v1; i is the same in every lane
__device__ __forceinline__ float logit_at(float v0, float v1, int i) { return __shfl_sync(0xffffffffu, i < 32 ? v0 : v1, i & 31); }

// The categorical head of row b (one warp): logits z = h_P W + b with lane l owning logits l and l + 32, one softmax per
// component (segmented warp reductions over a.coff), log-prob of the taken indices, entropy, and in MODE 1 the gradient
//   dz_ki = dlogp (1[i = a_k] - p_ki) + (entropy_scale / B) p_ki (log p_ki + H_k)
// into dpre [B,N] and the masked dh_P.  Every sum has a fixed order, so a repeated call is bit-identical.
template <int MODE>
__device__ __forceinline__ void cat_head_row(const HeadArgs& a, int b, int lane, float* vals) {
    const float* h = a.hp + (long long)b * a.Hp;
    const int N = a.N, K = a.A;
    const bool has0 = lane < N, has1 = lane + 32 < N;
    // logits: the rows of W are read coalesced, h 32 values at a time and broadcast lane to lane
    float z0 = 0.f, z1 = 0.f;
    for (int j0 = 0; j0 < a.Hp; j0 += 32) {
        const float hl = j0 + lane < a.Hp ? h[j0 + lane] : 0.f;
        const int n = a.Hp - j0 < 32 ? a.Hp - j0 : 32;
        for (int t = 0; t < n; ++t) {
            const float hj = __shfl_sync(0xffffffffu, hl, t);
            const float* w = a.wm + (long long)(j0 + t) * N;
            if (has0) z0 = fmaf(hj, w[lane], z0);
            if (has1) z1 = fmaf(hj, w[lane + 32], z1);
        }
    }
    if (has0) z0 += a.bm[lane];
    if (has1) z1 += a.bm[lane + 32];
    // component of each owned logit, and the per-component softmax: max, sum of exp, entropy (warp-uniform values)
    int c0 = 0, c1 = 0;
#pragma unroll
    for (int k = 1; k < kMaxActions; ++k)
        if (k < K) { c0 += lane >= a.coff[k]; c1 += lane + 32 >= a.coff[k]; }
    float mx[kMaxActions], lse[kMaxActions], ent[kMaxActions];
    float m0 = 0.f, m1 = 0.f, l0 = 0.f, l1 = 0.f, s0 = 1.f, s1 = 1.f, H0 = 0.f, H1 = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        float v = -INFINITY;
        if (has0 && c0 == k) v = z0;
        if (has1 && c1 == k) v = fmaxf(v, z1);
        mx[k] = warp_max(v);
        if (c0 == k) m0 = mx[k];
        if (c1 == k) m1 = mx[k];
    }
    const float e0 = has0 ? expf(z0 - m0) : 0.f, e1 = has1 ? expf(z1 - m1) : 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        const float s = warp_sum((c0 == k ? e0 : 0.f) + (c1 == k ? e1 : 0.f));
        lse[k] = logf(s);
        if (c0 == k) { l0 = lse[k]; s0 = s; }
        if (c1 == k) { l1 = lse[k]; s1 = s; }
    }
    const float lp0 = has0 ? z0 - m0 - l0 : 0.f, lp1 = has1 ? z1 - m1 - l1 : 0.f;   // log p
    const float p0 = e0 / s0, p1 = e1 / s1;
    float entropy = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        ent[k] = -warp_sum((c0 == k ? p0 * lp0 : 0.f) + (c1 == k ? p1 * lp1 : 0.f));
        entropy += ent[k];
        if (c0 == k) H0 = ent[k];
        if (c1 == k) H1 = ent[k];
    }
    (void)mx; (void)lse;
    if (MODE == 2) {
        float vsum = 0.f;
        const float* g = a.hv + (long long)b * a.Hv;
        for (int j = lane; j < a.Hv; j += 32) vsum = fmaf(g[j], a.wv[j], vsum);
        vsum = warp_sum(vsum);
        // greedy: the first largest logit; sampled: the first i with u < cumsum_i p (fp32, index order), else the last
        // index with p > 0.  Every lane runs the same scan on broadcast values; lane 0 writes.
        for (int k = 0; k < K; ++k) {
            const int lo = a.coff[k], hi = a.coff[k + 1];
            int pick = -1, last_pos = 0;
            if (a.noise == nullptr) {
                float best = -INFINITY;
                pick = 0;
                for (int i = lo; i < hi; ++i) {
                    const float zi = logit_at(z0, z1, i);
                    if (zi > best) { best = zi; pick = i - lo; }
                }
            } else {
                const float u = a.noise[(long long)b * K + k];
                float c = 0.f;
                for (int i = lo; i < hi; ++i) {
                    const float pi = logit_at(p0, p1, i);
                    c += pi;
                    if (pick < 0 && u < c) pick = i - lo;
                    if (pi > 0.f) last_pos = i - lo;
                }
                if (pick < 0) pick = last_pos;
            }
            if (lane == 0) a.action_out[(long long)b * K + k] = (float)pick;
        }
        if (lane == 0) a.v_out[b] = vsum + a.bv[0];
        return;
    }
    // log-prob of the taken indices (clamped into each component's range)
    const int row = a.idx != nullptr ? a.idx[b] : b;
    float logp = 0.f;
    int t0 = -1, t1 = -1;   // the taken index of the component of logit lane / lane + 32
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        const float av = a.actions[(long long)row * K + k];
        const int t = a.coff[k] + (int)fminf(fmaxf(av, 0.f), (float)(a.coff[k + 1] - a.coff[k] - 1));
        logp += logit_at(lp0, lp1, t);
        if (c0 == k) t0 = t;
        if (c1 == k) t1 = t;
    }
    if (MODE == 0) {
        if (lane == 0) a.logp_out[b] = logp;
        return;
    }
    const float* g = a.hv + (long long)b * a.Hv;
    float vsum = 0.f;
    for (int j = lane; j < a.Hv; j += 32) vsum = fmaf(g[j], a.wv[j], vsum);
    vsum = warp_sum(vsum);
    const float v = vsum + a.bv[0];
    const float logp_old = a.logp_old_in[a.logp_old_gathered ? row : b];
    const float ratio = expf(logp - logp_old);
    const float adv = a.adv[row], ret = a.returns[row];
    const float unclipped = ratio * adv;
    const float clipped = fminf(fmaxf(ratio, 1.f - a.eps_clip), 1.f + a.eps_clip) * adv;
    const float inv_b = 1.f / (float)a.B;
    const float dratio = unclipped <= clipped ? -adv * inv_b : 0.f;   // the Gaussian head's tf.minimum rule
    const float dlogp = dratio * ratio;
    const float dvv = a.value_scale * 2.f * inv_b * (v - ret);
    const float es = a.entropy_scale * inv_b;
    const float dz0 = has0 ? dlogp * ((lane == t0 ? 1.f : 0.f) - p0) + es * p0 * (lp0 + H0) : 0.f;
    const float dz1 = has1 ? dlogp * ((lane + 32 == t1 ? 1.f : 0.f) - p1) + es * p1 * (lp1 + H1) : 0.f;
    if (has0) a.dpre[(long long)b * N + lane] = dz0;
    if (has1) a.dpre[(long long)b * N + lane + 32] = dz1;
    if (lane == 0) {
        a.dv[b] = dvv;
        if (a.v_out != nullptr) a.v_out[b] = v;
    }
    // dh_P[j] = sum_i dz_i W[j, i] (i in index order), masked by h_P > 0; lane l owns j = j0 + l
    for (int j0 = 0; j0 < a.Hp; j0 += 32) {
        const int j = j0 + lane;
        const float* w = a.wm + (long long)(j < a.Hp ? j : 0) * N;
        float s = 0.f;
        for (int i = 0; i < N; ++i) s = fmaf(logit_at(dz0, dz1, i), w[i], s);
        if (j < a.Hp) a.dhp[(long long)b * a.Hp + j] = h[j] > 0.f ? s : 0.f;
    }
    for (int j = lane; j < a.Hv; j += 32) a.dhv[(long long)b * a.Hv + j] = g[j] > 0.f ? dvv * a.wv[j] : 0.f;
    vals[0] += fminf(unclipped, clipped);
    vals[1] += (v - ret) * (v - ret);
    vals[2] += ratio;
    vals[3] += entropy;
    if (a.kl_term) vals[7] += (ratio - 1.f) - (logp - logp_old);
}

// CAT: 0 = the Gaussian head, 1 = the categorical head
template <int MODE, int CAT>
__device__ __forceinline__ void head_row(const HeadArgs& a, int b, int lane, float* vals) {
    if constexpr (CAT != 0) cat_head_row<MODE>(a, b, lane, vals);
    else gauss_head_row<MODE>(a, b, lane, vals);
}

// CTA-level sum of the 8 warps' loss terms -> partial[block][8] (fixed order: deterministic)
__device__ __forceinline__ void head_block_reduce(const float* vals, float (*red)[8], float* partial_out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < 8; ++k) red[warp][k] = vals[k];
    __syncthreads();
    if (threadIdx.x < 8) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
        partial_out[threadIdx.x] = s;
    }
    __syncthreads();
}

// metrics[5] = policy_loss, value_loss, entropy_loss, loss, mean ratio; grads[logstd], value-bias etc.
// With guards, metrics rows are 7 wide: [5] = approx_kl (written here), [6] = the pre-clip gradient norm (written by the
// norm reduction); a minibatch evaluated after the stop gets a NaN row.
// CAT: the categorical head's entropy is the batch mean of slot 3 (sum_b H_b), and there is no logstd gradient.
template <int CAT>
__device__ __forceinline__ void ppo_finalize(const float* partial, int nblocks, int B, int A, const float* logstd, float value_scale,
                                             float entropy_scale, float* glogstd, float* metrics, float* tot /* shared [8] */,
                                             const Guards& g) {
    if (threadIdx.x < 8) {
        float s = 0.f;
        for (int i = 0; i < nblocks; ++i) s += __ldcg(partial + i * 8 + threadIdx.x);
        tot[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float inv_b = 1.f / (float)B;
        float ent = 0.f;
        if constexpr (CAT != 0) ent = tot[3] * inv_b;
        else
            for (int k = 0; k < A; ++k) {
                ent += kEntropyConst + logstd[k];
                glogstd[k] = tot[3 + k] - entropy_scale;
            }
        const float pl = tot[0] * inv_b;
        const float vl = tot[1] * inv_b * value_scale;
        const float el = ent * entropy_scale;
        if (g.stop != nullptr && __ldcg(g.stop) != 0u) {
            *g.stop = 2u;
            if (metrics != nullptr)
                for (int k = 0; k < 7; ++k) metrics[k] = __int_as_float(0x7fc00000);
        } else {
            if (metrics != nullptr) {
                metrics[0] = pl; metrics[1] = vl; metrics[2] = el; metrics[3] = -pl + vl - el; metrics[4] = tot[2] * inv_b;
            }
            if (g.stop != nullptr) {
                const float kl = tot[7] * inv_b;
                if (metrics != nullptr) metrics[5] = kl;
                if (g.kl_limit > 0.f && kl > g.kl_limit) *g.stop = 1u;
            }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// global L2 norm of the gradient (torch.nn.utils.clip_grad_norm_ over the 13 policy/ tensors; the layout's zero padding
// adds nothing).  Every sum has a fixed order, so a repeated call is bit-identical.
// ---------------------------------------------------------------------------------------------

// sum of v over the CTA's threads in a fixed order, returned to every thread; red: shared [blockDim.x / 32]
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    __syncthreads();                  // red may still be read by a previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

// this thread's share of sum(g^2): float4 elements k = first, first + stride, ...
__device__ __forceinline__ float sumsq_share(const float4* g, long long n4, long long first, long long stride) {
    float s = 0.f;
    for (long long k = first; k < n4; k += stride) {
        const float4 v = __ldcg(g + k);
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    }
    return s;
}

__device__ __forceinline__ float clip_coefficient(float sumsq, float max_norm) {
    if (max_norm <= 0.f) return 1.f;
    const float c = max_norm / (sqrtf(sumsq) + 1e-6f);
    return c < 1.f ? c : 1.f;
}

}  // namespace
}  // namespace cpb
