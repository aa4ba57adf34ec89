// What the PPO's files share: the launch-per-kernel path and the entry points' implementations (ppo.cu), the opt-in
// persistent learn() kernel (ppo_persistent.cu), GAE (gae.cu) and the C entry points (ppo_api.cu).  The functions declared
// below are hidden: the library's dynamic symbols stay the C ABI.
#pragma once
#include "common.cuh"

namespace cpb {

#pragma GCC visibility push(hidden)

constexpr int kMaxPpoDepth = 8;                          // hidden layers per trunk (cpb_ppo_spec)
constexpr int kMaxPpoTensors = 4 * kMaxPpoDepth + 5;
constexpr int kMaxActions = 4;
constexpr int kMaxLogits = 64;
constexpr int kMaxPersistentCtas = 1024;   // upper bound of the persistent learn() grid (one CTA per SM)

// Hidden-layer count and widths of trunk t (0: policy, 1: value) of a checked spec
__host__ __device__ __forceinline__ int trunk_depth(const cpb_ppo_spec& sp, int t) { return t ? sp.num_value : sp.num_policy; }
__host__ __device__ __forceinline__ int trunk_width(const cpb_ppo_spec& sp, int t, int l) {
    return t ? sp.value_sizes[l] : sp.policy_sizes[l];
}
// width of layer l's input: the state for layer 0
__host__ __device__ __forceinline__ int trunk_in(const cpb_ppo_spec& sp, int t, int l) {
    return l ? trunk_width(sp, t, l - 1) : sp.base.state_dim;
}
__host__ __device__ __forceinline__ int trunk_last(const cpb_ppo_spec& sp, int t) { return trunk_width(sp, t, trunk_depth(sp, t) - 1); }
__host__ __device__ __forceinline__ int max_depth(const cpb_ppo_spec& sp) {
    return sp.num_policy > sp.num_value ? sp.num_policy : sp.num_value;
}

// Tensors in TF creation order (ppo.py:38-66): policy layer l {kernel, bias} at 2l, the action head {action_mean/kernel,
// action_mean/bias, action_logstd} at 2P, value layer l at 2P + 3 + 2l, value/{kernel, bias} last.  Dense layers are
// named dense, dense_1, ... across both trunks in that order.
struct PpoLayout {
    int np, nv, n;
    int64_t off[kMaxPpoTensors], size[kMaxPpoTensors];
    int32_t shape[kMaxPpoTensors][2];
    int64_t total;
    __host__ __device__ int w(int t, int l) const { return t ? 2 * np + 3 + 2 * l : 2 * l; }
    __host__ __device__ int b(int t, int l) const { return w(t, l) + 1; }
    __host__ __device__ int wm() const { return 2 * np; }
    __host__ __device__ int bm() const { return 2 * np + 1; }
    __host__ __device__ int logstd() const { return 2 * np + 2; }
    __host__ __device__ int wv() const { return 2 * np + 3 + 2 * nv; }
    __host__ __device__ int bv() const { return wv() + 1; }
};

// The policy head of a plan.  Gaussian (cat == 0): N = K = num_actions columns of action_mean and an action_logstd.
// Categorical (cpb_ppo_cat_spec, cat == 1): N = sum n_k logits in action_logits, component k's at columns
// [off[k], off[k+1]); its layout keeps the logstd slot at size 0, so both kinds share PpoLayout's indexing.
struct HeadShape {
    int cat, K, N;
    int off[5];
};

// A categorical layout has no action_logstd: its public index i is PpoLayout's index i, or i + 1 past the head
__host__ __device__ __forceinline__ int cat_internal_index(const cpb_ppo_spec& sp, int i) { return i < 2 * sp.num_policy + 2 ? i : i + 1; }

// The per-call guards of the cpb_ppo_*_opts entry points (cpb_ppo_learn_options).  stop == nullptr on every other entry
// point: then none of the guard code runs and the metrics rows are 5 wide.
//   stop: device word, 0 while the update runs.  ppo_finalize sets it to 1 at the minibatch whose approx_kl exceeds
//         kl_limit and to 2 at every minibatch evaluated after that; Adam skips every step while it is non-zero.
//   clip: device float[1], the current minibatch's gradient scale min(1, max_norm / (norm + 1e-6)) (1 when max_norm == 0).
struct Guards {
    uint32_t* stop;
    float* clip;
    float* norm_partial;   // [kMaxPersistentCtas] per-block sums of squares of the gradient
    uint32_t* counter;     // blocks of grad_norm_kernel done (back to 0 when it ends)
    int32_t* steps;        // Adam steps applied (nullable)
    float max_norm;        // 0: no clipping
    float kl_limit;        // 1.5 * target_kl; 0: no stop
};

// ---------------------------------------------------------------------------------------------
// workspace plan
// ---------------------------------------------------------------------------------------------
struct PpoPlan {
    float* h[kMaxPpoDepth];    // layer l of both trunks: [B,Wp_l] policy then [B,Wv_l] value (a trunk past its depth: none)
    float* dh[kMaxPpoDepth];   // same shapes: masked gradients w.r.t. the layer outputs
    float* oh[kMaxPpoDepth];   // old-policy trunk [rows,Wp_l], l < P
    float *logp_old;       // [rows]
    float *dpre, *dv, *partial;
    float *ret32, *adv32;  // [T]
    double* gae_scratch;   // [T]
    float* norm_partial;   // [kMaxPersistentCtas]  guards of the options entry points (Guards)
    uint32_t* guard_words; // [4]: stop, counter, clip (as float bits), unused
    int64_t bytes;
    bool ok;
};

// width of trunk t's layer l, 0 past its depth
__host__ __device__ __forceinline__ int width_or_0(const cpb_ppo_spec& sp, int t, int l) {
    return l < trunk_depth(sp, t) ? trunk_width(sp, t, l) : 0;
}
// trunk t's part of a per-layer buffer (pl.h[l] / pl.dh[l]) at batch B
__host__ __device__ __forceinline__ float* trunk_buf(float* const* bufs, const cpb_ppo_spec& sp, int t, int l, int B) {
    return bufs[l] + (t ? (long long)B * width_or_0(sp, 0, l) : 0);
}

// ---- ppo.cu: the spec checks, the layout and the plan, and the (spec, head shape) implementations of the entry points
int32_t check_ppo_spec(const cpb_ppo_spec* sp);
HeadShape gauss_head(const cpb_ppo_spec* sp);
int32_t cat_head(const cpb_ppo_cat_spec* cs, HeadShape* hs);
const char* ppo_tensor_name(const cpb_ppo_spec* sp, int i);
PpoPlan make_ppo_plan(void* ws, int64_t ws_bytes, const cpb_ppo_spec* sp, const HeadShape& hs, int max_batch, int horizon);

int32_t ppo_layout(const cpb_ppo_spec* spec, const HeadShape& hs, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                   int64_t* total);
int32_t ppo_forward(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* states, int32_t batch,
                    const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes, void* stream);
int32_t ppo_loss_grad(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* params_old,
                      const float* states, const float* actions, const float* returns, const float* advantages,
                      const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                      int64_t workspace_bytes, void* stream);
int32_t ppo_train_step(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old, float* grads,
                       float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                       const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                       int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream);
int32_t ppo_train_step_opts(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old,
                            float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                            const float* states, const float* actions, const float* returns, const float* advantages,
                            const int32_t* idx, int32_t batch, float* metrics, const cpb_ppo_learn_options* opts,
                            uint32_t* stop, int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);
// learn and its options twin (guarded: opts / steps_applied are used and the metrics rows are 7 wide)
int32_t ppo_learn(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old, float* grads,
                  float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                  const float* actions, const double* rewards, const double* values, double bootstrap_value,
                  const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                  const int32_t* perms, float* metrics, bool guarded, const cpb_ppo_learn_options* opts,
                  int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);
// learn_segments and its options twin
int32_t ppo_learn_segments(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old, float* grads,
                           float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, const double* bootstrap_values,
                           const double* dones, const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                           double gamma, double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                           float* metrics, bool guarded, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                           void* workspace, int64_t workspace_bytes, void* stream);

// ---- ppo_persistent.cu: the opt-in (CPB_PPO_PERSISTENT=1) persistent cooperative kernel that runs all num_epochs x nmb
// minibatch steps of learn() in one launch.  *launched is false when it is off, unavailable or num_epochs == 0: the
// caller then runs the launch-per-kernel steps.
int32_t learn_persistent(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, float* params,
                         float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                         const float* states, const float* actions, int T, int num_epochs, int batch_size, int nmb,
                         const int32_t* perms, float* metrics, const Guards& gd, cudaStream_t s, bool* launched);

// ---- gae.cu: GAE of one rollout (gae_kernel) and over segments; each output may be null, adv_out null needs `scratch` [T]
int32_t launch_gae(const double* rewards, const double* values, double bootstrap, const double* dones, int T, double gamma,
                   double lam, double* adv_out, double* ret_out, double* advn_out, float* ret32, float* advn32,
                   double* scratch, cudaStream_t s);
int32_t launch_gae_segments(const double* rewards, const double* values, const double* bootstrap, const double* dones,
                            const int32_t* offsets, int num_segments, int rows, double gamma, double lam, double* adv,
                            double* ret_out, double* advn_out, float* ret32, float* advn32, cudaStream_t s);

#pragma GCC visibility pop

}  // namespace cpb
