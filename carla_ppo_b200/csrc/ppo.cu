// PPO update path behind the C ABI: Gaussian-policy / value MLPs (reference ppo.py:38-66), clipped
// surrogate + value + entropy loss and its gradient (ppo.py:119-144) and the driver's update block (train.py:171-207),
// one kernel launch per step.  Everything here is latency-bound (369 505 parameters, minibatches of a few hundred rows):
// the kernels are small bounds-checked fp32 tile GEMMs, batched over the two trunks (policy / value) so one minibatch step
// is ~11 launches with no host sync.  The C entry points are in ppo_api.cu, GAE in gae.cu and the opt-in persistent
// learn() kernel in ppo_persistent.cu.
#include <cmath>

#include "elementwise.cuh"
#include "ppo_device.cuh"

namespace cpb {

namespace {

PpoLayout make_ppo_layout(const cpb_ppo_spec* sp, const HeadShape& hs) {
    PpoLayout L;
    memset(&L, 0, sizeof(L));
    const int A = sp->base.num_actions;
    L.np = sp->num_policy; L.nv = sp->num_value; L.n = 2 * (L.np + L.nv) + 5;
    auto set = [&](int i, int rows, int cols) { L.shape[i][0] = rows; L.shape[i][1] = cols; };
    for (int t = 0; t < 2; ++t)
        for (int l = 0; l < trunk_depth(*sp, t); ++l) {
            set(L.w(t, l), trunk_in(*sp, t, l), trunk_width(*sp, t, l));
            set(L.b(t, l), trunk_width(*sp, t, l), 0);
        }
    if (hs.cat) { set(L.wm(), trunk_last(*sp, 0), hs.N); set(L.bm(), hs.N, 0); }
    else { set(L.wm(), trunk_last(*sp, 0), A); set(L.bm(), A, 0); set(L.logstd(), A, 0); }
    set(L.wv(), trunk_last(*sp, 1), 1); set(L.bv(), 1, 0);
    int64_t o = 0;
    for (int i = 0; i < L.n; ++i) {
        L.size[i] = (int64_t)L.shape[i][0] * (L.shape[i][1] ? L.shape[i][1] : 1);
        L.off[i] = o;
        o += align_up(L.size[i], 64);
    }
    L.total = o;
    return L;
}

template <int GATHER>
__global__ void __launch_bounds__(kTileThreads)
small_gemm_kernel(const __grid_constant__ GemmBatch batch) {
    const GemmJob& J = batch.job[blockIdx.z];
    const int m0 = blockIdx.x * TS, n0 = blockIdx.y * TS;
    if (m0 >= J.M || n0 >= J.N) return;
    // double-buffered tiles: the global loads of chunk i+1 are in flight (in registers) while chunk i is multiplied
    __shared__ __align__(16) float As[2][TK][TS + 4];
    __shared__ __align__(16) float Bs[2][TK][TS + 4];
    gemm_tile<GATHER>(J, m0, n0, blockIdx.x == 0, threadIdx.x, As, Bs, [] { __syncthreads(); });
}

int32_t launch_small_gemm(const GemmBatch& b, int njobs, cudaStream_t s) {
    int maxM = 0, maxN = 0;
    for (int i = 0; i < njobs; ++i) {
        if (b.job[i].M > maxM) maxM = b.job[i].M;
        if (b.job[i].N > maxN) maxN = b.job[i].N;
    }
    if (maxM == 0 || maxN == 0) return CPB_OK;
    dim3 grid(cdiv(maxM, TS), cdiv(maxN, TS), njobs);
    const int gather = b.job[0].a.gather == nullptr ? 0 : (b.job[0].a.gather_on_o ? 1 : 2);   // same for all jobs of a batch
    if (gather == 0) small_gemm_kernel<0><<<grid, kTileThreads, 0, s>>>(b);
    else if (gather == 1) small_gemm_kernel<1><<<grid, kTileThreads, 0, s>>>(b);
    else small_gemm_kernel<2><<<grid, kTileThreads, 0, s>>>(b);
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int MODE, int CAT>
__global__ void __launch_bounds__(256)
ppo_head_kernel(const __grid_constant__ HeadArgs a) {
    __shared__ float red[8][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    float vals[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (b < a.B) head_row<MODE, CAT>(a, b, lane, vals);
    if (MODE == 1) head_block_reduce(vals, red, a.partial + blockIdx.x * 8);
}

template <int MODE>
void launch_head(const HeadShape& hs, int B, const HeadArgs& h, cudaStream_t s) {
    if (hs.cat) ppo_head_kernel<MODE, 1><<<cdiv(B, 8), 256, 0, s>>>(h);
    else ppo_head_kernel<MODE, 0><<<cdiv(B, 8), 256, 0, s>>>(h);
}

template <int CAT>
__global__ void ppo_finalize_kernel(const float* __restrict__ partial, int nblocks, int B, int A,
                                    const float* __restrict__ logstd, float value_scale, float entropy_scale,
                                    float* __restrict__ glogstd, float* __restrict__ metrics, const Guards g) {
    __shared__ float tot[8];
    ppo_finalize<CAT>(partial, nblocks, B, A, logstd, value_scale, entropy_scale, glogstd, metrics, tot, g);
}

constexpr int kNormBlocks = 256, kNormThreads = 256;

// partial sums per block, then the last block to finish sums the partials in block order: clip coefficient, metrics[6]
__global__ void __launch_bounds__(kNormThreads)
grad_norm_kernel(const float4* __restrict__ g, long long n4, const Guards gd, float* __restrict__ metrics) {
    __shared__ float red[kNormThreads / 32];
    __shared__ bool last;
    const float s = block_sum(sumsq_share(g, n4, (long long)blockIdx.x * blockDim.x + threadIdx.x, (long long)gridDim.x * blockDim.x), red);
    if (threadIdx.x == 0) {
        gd.norm_partial[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(gd.counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    float t = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(gd.norm_partial + i);
    t = block_sum(t, red);
    if (threadIdx.x == 0) {
        gd.clip[0] = clip_coefficient(t, gd.max_norm);
        if (metrics != nullptr && __ldcg(gd.stop) != 2u) metrics[6] = sqrtf(t);
        *gd.counter = 0u;
    }
}

int32_t launch_grad_norm(const float* grads, long long n, const Guards& gd, float* metrics, cudaStream_t s) {
    grad_norm_kernel<<<kNormBlocks, kNormThreads, 0, s>>>(reinterpret_cast<const float4*>(grads), n / 4, gd, metrics);
    CPB_LAUNCHED();
    return CPB_OK;
}

// log pi_old(a|s) for `rows` samples (optionally gathered)
int32_t run_old_logp(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, const float* params_old,
                     const float* states, const float* actions, const int32_t* idx, int rows, cudaStream_t s) {
    GemmBatch gb;
    for (int l = 0; l < sp->num_policy; ++l) {
        gb.job[0] = fwd_job(l ? pl.oh[l - 1] : states, l ? nullptr : idx, rows, trunk_in(*sp, 0, l),
                            params_old + L.off[L.w(0, l)], sp->policy_sizes[l], params_old + L.off[L.b(0, l)], pl.oh[l], 1);
        CPB_TRY(launch_small_gemm(gb, 1, s));
    }
    HeadArgs h = head_args(*sp, hs, L, params_old, rows);
    h.hp = pl.oh[sp->num_policy - 1]; h.actions = actions; h.idx = idx; h.logp_out = pl.logp_old;
    launch_head<0>(hs, rows, h, s);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t run_trunks(const cpb_ppo_spec* sp, const PpoLayout& L, const PpoPlan& pl, const float* params,
                   const float* states, const int32_t* idx, int B, cudaStream_t s) {
    GemmBatch gb;
    for (int l = 0; l < max_depth(*sp); ++l)
        CPB_TRY(launch_small_gemm(gb, trunk_fwd_jobs(*sp, L, pl, params, states, idx, B, l, gb.job), s));
    return CPB_OK;
}

// forward + loss + gradients for one minibatch; logp_old given (gathered or not)
int32_t run_loss_grad(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, const float* params,
                      const float* states, const float* actions, const float* returns, const float* adv,
                      const int32_t* idx, int B, const float* logp_old, int logp_old_gathered, float* grads,
                      float* metrics, const Guards& gd, cudaStream_t s) {
    const cpb_ppo_config* c = &sp->base;
    const int P = sp->num_policy, V = sp->num_value, D = max_depth(*sp);
    CPB_TRY(run_trunks(sp, L, pl, params, states, idx, B, s));
    HeadArgs h = head_args(*sp, hs, L, params, B);
    h.hp = trunk_buf(pl.h, *sp, 0, P - 1, B); h.hv = trunk_buf(pl.h, *sp, 1, V - 1, B);
    h.actions = actions; h.returns = returns; h.adv = adv; h.idx = idx;
    h.logp_old_in = logp_old; h.logp_old_gathered = logp_old_gathered;
    h.dpre = pl.dpre; h.dv = pl.dv; h.dhp = trunk_buf(pl.dh, *sp, 0, P - 1, B); h.dhv = trunk_buf(pl.dh, *sp, 1, V - 1, B);
    h.partial = pl.partial;
    h.kl_term = gd.stop != nullptr;
    const int nblocks = cdiv(B, 8);
    launch_head<1>(hs, B, h, s);
    CPB_LAUNCHED();
    if (hs.cat)
        ppo_finalize_kernel<1><<<1, 32, 0, s>>>(pl.partial, nblocks, B, c->num_actions, nullptr, c->value_scale,
                                                c->entropy_scale, nullptr, metrics, gd);
    else
        ppo_finalize_kernel<0><<<1, 32, 0, s>>>(pl.partial, nblocks, B, c->num_actions, params + L.off[L.logstd()],
                                                c->value_scale, c->entropy_scale, grads + L.off[L.logstd()], metrics, gd);
    CPB_LAUNCHED();
    // one launch per layer, top down, for both trunks: weight gradients and the data gradient into the layer below.  The
    // head weight gradients only need the head kernel's outputs and join the top layer's launch (at two layers per trunk:
    // 6 independent GEMMs), unless that launch gathers the states (one layer in both trunks).
    GemmBatch gb;
    for (int l = D - 1; l >= 0; --l) {
        int n = trunk_bwd_jobs(*sp, L, pl, params, grads, states, idx, B, l, gb.job);
        if (l == D - 1) {
            if (l == 0 && idx != nullptr) {
                GemmBatch hb;
                head_bwd_jobs(*sp, L, pl, grads, B, hs.N, hb.job);
                CPB_TRY(launch_small_gemm(hb, 2, s));
            } else {
                head_bwd_jobs(*sp, L, pl, grads, B, hs.N, gb.job + n);
                n += 2;
            }
        }
        CPB_TRY(launch_small_gemm(gb, n, s));
    }
    return CPB_OK;
}

// Everything of the driver's update block after GAE (train.py:178-207): theta_old <- theta, the old policy's
// log-probabilities, and num_epochs x ceil(T / batch_size) minibatch Adam steps reading pl.ret32 / pl.adv32.
int32_t learn_update(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, float* params, float* params_old,
                     float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                     const float* states, const float* actions, int T, int num_epochs, int batch_size,
                     const int32_t* perms, float* metrics, const Guards& gd, cudaStream_t s) {
    const int mcols = gd.stop != nullptr ? 7 : 5;
    // theta_old <- theta (PPO.update_old_policy, ppo.py:275-276)
    CPB_CUDA(cudaMemcpyAsync(params_old, params, L.total * sizeof(float), cudaMemcpyDeviceToDevice, s));
    // log pi_old(a_t|s_t) is constant during the update: evaluate it once for all T samples
    CPB_TRY(run_old_logp(sp, hs, L, pl, params_old, states, actions, nullptr, T, s));
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    const int nmb = cdiv(T, batch_size);
    bool launched = false;
    CPB_TRY(learn_persistent(sp, hs, L, pl, params, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, T, num_epochs,
                             batch_size, nmb, perms, metrics, gd, s, &launched));
    if (launched) return CPB_OK;
    for (int e = 0; e < num_epochs; ++e)
        for (int i = 0; i < nmb; ++i) {
            const int begin = i * batch_size;
            const int B = begin + batch_size <= T ? batch_size : T - begin;
            const int32_t* idx = perms + (long long)e * T + begin;
            float* mt = metrics ? metrics + ((long long)e * nmb + i) * mcols : nullptr;
            CPB_TRY(run_loss_grad(sp, hs, L, pl, params, states, actions, pl.ret32, pl.adv32, idx, B, pl.logp_old, 1,
                                  grads, mt, gd, s));
            if (gd.stop != nullptr) {
                // the minibatches after a stop are still launched (the host cannot know); Adam skips them on the device
                CPB_TRY(launch_grad_norm(grads, L.total, gd, mt, s));
                CPB_TRY(launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s,
                                    gd.stop, gd.clip, gd.steps));
            } else {
                CPB_TRY(launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s));
            }
        }
    return CPB_OK;
}

// cpb_ppo_learn_options -> Guards on the plan's guard scratch, refusing bad options before anything is enqueued.  stop:
// the caller's stop word (train_step), or null for a zeroed word of the call's own (learn).  steps_applied is zeroed.
int32_t make_guards(const cpb_ppo_learn_options* opts, const PpoPlan& pl, uint32_t* stop, int32_t* steps_applied,
                    cudaStream_t s, Guards* gd) {
    float max_norm = 0.f, target_kl = 0.f;
    if (opts != nullptr) { max_norm = opts->max_grad_norm; target_kl = opts->target_kl; }
    CPB_REQUIRE(std::isfinite(max_norm) && max_norm >= 0.f, "ppo options: max_grad_norm must be finite and >= 0 (0 = off)");
    CPB_REQUIRE(std::isfinite(target_kl) && target_kl >= 0.f, "ppo options: target_kl must be finite and >= 0 (0 = off)");
    memset(gd, 0, sizeof(*gd));
    gd->stop = stop != nullptr ? stop : pl.guard_words;
    gd->counter = pl.guard_words + 1;
    gd->clip = reinterpret_cast<float*>(pl.guard_words + 2);
    gd->norm_partial = pl.norm_partial;
    gd->steps = steps_applied;
    gd->max_norm = max_norm;
    gd->kl_limit = (float)(1.5 * (double)target_kl);
    // the plan's own stop word (used when the caller gives none) and the norm reduction's block counter start at 0
    CPB_CUDA(cudaMemsetAsync(pl.guard_words, 0, 2 * sizeof(uint32_t), s));
    if (steps_applied != nullptr) CPB_CUDA(cudaMemsetAsync(steps_applied, 0, sizeof(int32_t), s));
    return CPB_OK;
}

}  // namespace

HeadShape gauss_head(const cpb_ppo_spec* sp) {
    HeadShape hs;
    memset(&hs, 0, sizeof(hs));
    hs.K = hs.N = sp->base.num_actions;
    return hs;
}

const char* ppo_tensor_name(const cpb_ppo_spec* sp, int i) {
    static char dense[2 * kMaxPpoDepth][2][24];
    static const bool ready = [] {
        for (int k = 0; k < 2 * kMaxPpoDepth; ++k)
            for (int b = 0; b < 2; ++b) {
                char suffix[8] = "";
                if (k) snprintf(suffix, sizeof(suffix), "_%d", k);
                snprintf(dense[k][b], sizeof(dense[k][b]), "dense%s/%s", suffix, b ? "bias" : "kernel");
            }
        return true;
    }();
    (void)ready;
    static const char* heads[5] = {"action_mean/kernel", "action_mean/bias", "action_logstd", "value/kernel", "value/bias"};
    const int P = sp->num_policy, V = sp->num_value;
    if (i < 0 || i >= 2 * (P + V) + 5) return nullptr;
    if (i < 2 * P) return dense[i / 2][i % 2];
    if (i < 2 * P + 3) return heads[i - 2 * P];
    if (i < 2 * P + 3 + 2 * V) return dense[P + (i - 2 * P - 3) / 2][(i - 2 * P - 3) % 2];
    return heads[3 + i - (2 * P + 3 + 2 * V)];
}

PpoPlan make_ppo_plan(void* ws, int64_t ws_bytes, const cpb_ppo_spec* sp, const HeadShape& hs, int max_batch, int horizon) {
    PpoPlan p;
    memset(&p, 0, sizeof(p));
    Arena a(ws, ws_bytes);
    const int64_t B = max_batch;
    const int64_t rows = horizon > max_batch ? horizon : max_batch;
    const int D = max_depth(*sp);
    for (int l = 0; l < D; ++l) p.h[l] = a.take<float>(B * (width_or_0(*sp, 0, l) + width_or_0(*sp, 1, l)));
    for (int l = D - 1; l >= 0; --l) p.dh[l] = a.take<float>(B * (width_or_0(*sp, 0, l) + width_or_0(*sp, 1, l)));
    for (int l = 0; l < sp->num_policy; ++l) p.oh[l] = a.take<float>(rows * sp->policy_sizes[l]);
    p.logp_old = a.take<float>(rows);
    p.dpre = a.take<float>(B * (hs.cat ? hs.N : kMaxActions));
    p.dv = a.take<float>(B);
    p.partial = a.take<float>((int64_t)(cdiv(B, 8) > kMaxPersistentCtas ? cdiv(B, 8) : kMaxPersistentCtas) * 8);
    p.ret32 = a.take<float>(rows);
    p.adv32 = a.take<float>(rows);
    p.gae_scratch = a.take<double>(rows);
    p.norm_partial = a.take<float>(kMaxPersistentCtas);
    p.guard_words = a.take<uint32_t>(4);
    p.bytes = a.off;
    p.ok = ws == nullptr || !a.overflow;
    return p;
}

int32_t check_ppo_spec(const cpb_ppo_spec* sp) {
    CPB_REQUIRE(sp != nullptr, "ppo spec is NULL");
    const cpb_ppo_config* c = &sp->base;
    CPB_REQUIRE(c->hidden1 == 0 && c->hidden2 == 0,
                "ppo spec: base.hidden1 / base.hidden2 must be 0 (the widths are policy_sizes / value_sizes), got %d, %d",
                c->hidden1, c->hidden2);
    CPB_REQUIRE(c->state_dim >= 1, "ppo: state_dim must be >= 1, got %d", c->state_dim);
    CPB_REQUIRE(c->num_actions >= 1 && c->num_actions <= kMaxActions, "ppo: num_actions must be in [1,%d]", kMaxActions);
    CPB_REQUIRE(sp->num_policy >= 1 && sp->num_policy <= kMaxPpoDepth && sp->num_value >= 1 && sp->num_value <= kMaxPpoDepth,
                "ppo spec: each trunk needs 1 to %d hidden layers, got %d (policy) and %d (value)", kMaxPpoDepth,
                sp->num_policy, sp->num_value);
    for (int t = 0; t < 2; ++t)
        for (int l = 0; l < trunk_depth(*sp, t); ++l)
            CPB_REQUIRE(trunk_width(*sp, t, l) >= 1, "ppo spec: %s layer %d has width %d (must be >= 1)",
                        t ? "value" : "policy", l, trunk_width(*sp, t, l));
    return CPB_OK;
}

// A cpb_ppo_cat_spec -> its HeadShape, refusing a bad one (the Gaussian spec's checks first)
int32_t cat_head(const cpb_ppo_cat_spec* cs, HeadShape* hs) {
    CPB_REQUIRE(cs != nullptr, "ppo categorical spec is NULL");
    CPB_TRY(check_ppo_spec(&cs->spec));
    const cpb_ppo_config& c = cs->spec.base;
    for (int k = 0; k < kMaxActions; ++k)
        CPB_REQUIRE(c.action_low[k] == 0.f && c.action_high[k] == 0.f,
                    "ppo categorical spec: spec.base.action_low / action_high must be 0 (component %d)", k);
    memset(hs, 0, sizeof(*hs));
    hs->cat = 1;
    hs->K = c.num_actions;
    for (int k = 0; k < hs->K; ++k) {
        const int n = cs->num_categories[k];
        CPB_REQUIRE(n >= 2 && n <= kMaxLogits, "ppo categorical spec: component %d has %d categories (must be 2..%d)", k, n,
                    kMaxLogits);
        hs->off[k + 1] = hs->off[k] + n;
    }
    hs->N = hs->off[hs->K];
    for (int k = hs->K + 1; k < 5; ++k) hs->off[k] = hs->N;
    CPB_REQUIRE(hs->N <= kMaxLogits, "ppo categorical spec: %d logits in all (at most %d)", hs->N, kMaxLogits);
    return CPB_OK;
}

#define CPB_PPO_PLAN(maxb, horizon)                                                            \
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");                                    \
    PpoPlan pl = make_ppo_plan(workspace, workspace_bytes, spec, hs, maxb, horizon);           \
    if (!pl.ok) {                                                                              \
        cpb::set_error("ppo workspace too small: need %lld bytes, got %lld", (long long)pl.bytes, \
                       (long long)workspace_bytes);                                            \
        return CPB_ERR_WORKSPACE_TOO_SMALL;                                                    \
    }                                                                                          \
    PpoLayout L = make_ppo_layout(spec, hs);                                                   \
    cudaStream_t s = (cudaStream_t)stream;

int32_t ppo_layout(const cpb_ppo_spec* spec, const HeadShape& hs, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                   int64_t* total) {
    PpoLayout L = make_ppo_layout(spec, hs);
    const int n = hs.cat ? L.n - 1 : L.n;
    for (int e = 0; e < n; ++e) {
        const int i = hs.cat ? cat_internal_index(*spec, e) : e;
        if (offsets) offsets[e] = L.off[i];
        if (sizes) sizes[e] = L.size[i];
        if (shapes) { shapes[e * 2] = L.shape[i][0]; shapes[e * 2 + 1] = L.shape[i][1]; }
    }
    if (total) *total = L.total;
    return CPB_OK;
}

int32_t ppo_forward(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* states, int32_t batch,
                    const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                    void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_forward: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && states && action && value, "ppo_forward: NULL pointer");
    CPB_TRY(run_trunks(spec, L, pl, params, states, nullptr, batch, s));
    HeadArgs h = head_args(*spec, hs, L, params, batch);
    h.hp = trunk_buf(pl.h, *spec, 0, spec->num_policy - 1, batch); h.hv = trunk_buf(pl.h, *spec, 1, spec->num_value - 1, batch);
    h.noise = noise; h.action_out = action; h.v_out = value;
    launch_head<2>(hs, batch, h, s);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t ppo_loss_grad(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* params_old,
                      const float* states, const float* actions, const float* returns, const float* advantages,
                      const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                      int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_loss_grad: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && params_old && states && actions && returns && advantages && grads, "ppo_loss_grad: NULL pointer");
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    CPB_TRY(run_old_logp(spec, hs, L, pl, params_old, states, actions, idx, batch, s));
    return run_loss_grad(spec, hs, L, pl, params, states, actions, returns, advantages, idx, batch, pl.logp_old, 0, grads,
                         metrics, Guards{}, s);
}

int32_t ppo_train_step(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old, float* grads,
                       float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                       const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                       int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(lr_dev != nullptr, "ppo_train_step: lr_dev is NULL");
    CPB_TRY(ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                          workspace, workspace_bytes, stream));
    PpoLayout L = make_ppo_layout(spec, hs);
    return launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f,
                       (cudaStream_t)stream);
}

int32_t ppo_train_step_opts(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old,
                            float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                            const float* states, const float* actions, const float* returns, const float* advantages,
                            const int32_t* idx, int32_t batch, float* metrics, const cpb_ppo_learn_options* opts,
                            uint32_t* stop, int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_train_step_opts: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                returns && advantages, "ppo_train_step_opts: NULL pointer");
    Guards gd;
    CPB_TRY(make_guards(opts, pl, stop, steps_applied, s, &gd));
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    CPB_TRY(run_old_logp(spec, hs, L, pl, params_old, states, actions, idx, batch, s));
    CPB_TRY(run_loss_grad(spec, hs, L, pl, params, states, actions, returns, advantages, idx, batch, pl.logp_old, 0, grads,
                          metrics, gd, s));
    CPB_TRY(launch_grad_norm(grads, L.total, gd, metrics, s));
    return launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s, gd.stop,
                       gd.clip, gd.steps);
}

int32_t ppo_learn(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old, float* grads,
                  float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                  const float* actions, const double* rewards, const double* values, double bootstrap_value,
                  const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                  const int32_t* perms, float* metrics, bool guarded, const cpb_ppo_learn_options* opts,
                  int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(T >= 1 && batch_size >= 1 && num_epochs >= 0, "ppo_learn: bad sizes");
    CPB_PPO_PLAN(batch_size < T ? batch_size : T, T);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                rewards && values && dones, "ppo_learn: NULL pointer");
    CPB_REQUIRE(perms != nullptr || num_epochs == 0, "ppo_learn: perms is NULL");
    Guards gd{};
    if (guarded) CPB_TRY(make_guards(opts, pl, nullptr, steps_applied, s, &gd));
    // GAE, returns, normalised advantages (float64), rounded to float32 like the reference's feed
    CPB_TRY(launch_gae(rewards, values, bootstrap_value, dones, T, gamma, lam, nullptr, nullptr, nullptr, pl.ret32, pl.adv32,
                       pl.gae_scratch, s));
    return learn_update(spec, hs, L, pl, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, T,
                        num_epochs, batch_size, perms, metrics, gd, s);
}

int32_t ppo_learn_segments(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old, float* grads,
                           float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, const double* bootstrap_values,
                           const double* dones, const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                           double gamma, double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                           float* metrics, bool guarded, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                           void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(num_segments >= 1 && rows >= num_segments && batch_size >= 1 && num_epochs >= 0,
                "ppo_learn_segments: bad sizes");
    CPB_PPO_PLAN(batch_size < rows ? batch_size : rows, rows);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                rewards && values && bootstrap_values && dones && segment_offsets, "ppo_learn_segments: NULL pointer");
    CPB_REQUIRE(perms != nullptr || num_epochs == 0, "ppo_learn_segments: perms is NULL");
    Guards gd{};
    if (guarded) CPB_TRY(make_guards(opts, pl, nullptr, steps_applied, s, &gd));
    // GAE per segment, then returns and advantages normalised over all rows (float64), rounded to float32
    CPB_TRY(launch_gae_segments(rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                                pl.gae_scratch, nullptr, nullptr, pl.ret32, pl.adv32, s));
    return learn_update(spec, hs, L, pl, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rows,
                        num_epochs, batch_size, perms, metrics, gd, s);
}

}  // namespace cpb
