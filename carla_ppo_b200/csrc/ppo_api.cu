// The PPO's C entry points (GAE's are in gae.cu): the cpb_ppo_spec ones, their cpb_ppo_cat_spec twins and the two-per-side
// cpb_ppo_config ones.  Each checks its spec and calls the (spec, head shape) implementation in ppo.cu.
#include "ppo.cuh"

using namespace cpb;

constexpr int kLegacyPpoTensors = 13;                     // two layers per trunk (cpb_ppo_config)

extern "C" {

int32_t cpb_ppo_num_tensors(void) { return kLegacyPpoTensors; }
const char* cpb_ppo_tensor_name(int32_t i) {
    cpb_ppo_spec sp;
    memset(&sp, 0, sizeof(sp));
    sp.num_policy = sp.num_value = 2;
    return ppo_tensor_name(&sp, i);
}

int32_t cpb_ppo_spec_num_tensors(const cpb_ppo_spec* spec) {
    CPB_TRY(check_ppo_spec(spec));
    return 2 * (spec->num_policy + spec->num_value) + 5;
}
const char* cpb_ppo_spec_tensor_name(const cpb_ppo_spec* spec, int32_t i) {
    if (check_ppo_spec(spec) != CPB_OK) return nullptr;
    return ppo_tensor_name(spec, i);
}

int32_t cpb_ppo_spec_layout(const cpb_ppo_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_TRY(check_ppo_spec(spec));
    return ppo_layout(spec, gauss_head(spec), offsets, sizes, shapes, total);
}

int64_t cpb_ppo_spec_workspace_bytes(const cpb_ppo_spec* spec, int32_t max_batch, int32_t horizon) {
    if (check_ppo_spec(spec) != CPB_OK || max_batch < 1 || horizon < 0) return CPB_ERR_INVALID_ARGUMENT;
    return make_ppo_plan(nullptr, 0, spec, gauss_head(spec), max_batch, horizon).bytes;
}

// the cpb_ppo_spec_* entry points: check the spec, then the shared implementation with the Gaussian head
#define CPB_PPO_GAUSS()              \
    CPB_TRY(check_ppo_spec(spec));   \
    const HeadShape hs = gauss_head(spec);

int32_t cpb_ppo_spec_forward(const cpb_ppo_spec* spec, const float* params, const float* states, int32_t batch,
                             const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                             void* stream) {
    CPB_PPO_GAUSS();
    return ppo_forward(spec, hs, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_loss_grad(const cpb_ppo_spec* spec, const float* params, const float* params_old,
                               const float* states, const float* actions, const float* returns, const float* advantages,
                               const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                         workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_train_step(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                                const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                                int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_train_step(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, returns,
                          advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_train_step_opts(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                     float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                     const float* states, const float* actions, const float* returns,
                                     const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                     const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_train_step_opts(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                               returns, advantages, idx, batch, metrics, opts, stop, steps_applied, workspace,
                               workspace_bytes, stream);
}

int32_t cpb_ppo_spec_learn(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, double bootstrap_value,
                           const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                           int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, false, nullptr,
                     nullptr, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_learn_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                                const float* actions, const double* rewards, const double* values, double bootstrap_value,
                                const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                                int32_t batch_size, const int32_t* perms, float* metrics,
                                const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                                int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, true, opts,
                     steps_applied, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_learn_segments(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                    double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                    float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, false, nullptr, nullptr, workspace, workspace_bytes,
                              stream);
}

int32_t cpb_ppo_spec_learn_segments_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                         float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                         const float* states, const float* actions, const double* rewards,
                                         const double* values, const double* bootstrap_values, const double* dones,
                                         const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                         double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                         float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, true, opts, steps_applied, workspace,
                              workspace_bytes, stream);
}

// ---- The categorical twins: check the cpb_ppo_cat_spec, then the shared implementation with its head
#define CPB_PPO_CAT()                 \
    HeadShape hs;                     \
    CPB_TRY(cat_head(cspec, &hs));    \
    const cpb_ppo_spec* spec = &cspec->spec;

int32_t cpb_ppo_cat_num_tensors(const cpb_ppo_cat_spec* cspec) {
    CPB_PPO_CAT();
    return 2 * (spec->num_policy + spec->num_value) + 4;
}
const char* cpb_ppo_cat_tensor_name(const cpb_ppo_cat_spec* cspec, int32_t i) {
    HeadShape hs;
    if (cat_head(cspec, &hs) != CPB_OK) return nullptr;
    const cpb_ppo_spec* spec = &cspec->spec;
    if (i < 0 || i >= 2 * (spec->num_policy + spec->num_value) + 4) return nullptr;
    const int k = cat_internal_index(*spec, i);
    if (k == 2 * spec->num_policy) return "action_logits/kernel";
    if (k == 2 * spec->num_policy + 1) return "action_logits/bias";
    return ppo_tensor_name(spec, k);
}
int32_t cpb_ppo_cat_layout(const cpb_ppo_cat_spec* cspec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_PPO_CAT();
    return ppo_layout(spec, hs, offsets, sizes, shapes, total);
}
int64_t cpb_ppo_cat_workspace_bytes(const cpb_ppo_cat_spec* cspec, int32_t max_batch, int32_t horizon) {
    HeadShape hs;
    if (cat_head(cspec, &hs) != CPB_OK || max_batch < 1 || horizon < 0) return CPB_ERR_INVALID_ARGUMENT;
    return make_ppo_plan(nullptr, 0, &cspec->spec, hs, max_batch, horizon).bytes;
}

int32_t cpb_ppo_cat_forward(const cpb_ppo_cat_spec* cspec, const float* params, const float* states, int32_t batch,
                            const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                            void* stream) {
    CPB_PPO_CAT();
    return ppo_forward(spec, hs, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_loss_grad(const cpb_ppo_cat_spec* cspec, const float* params, const float* params_old,
                              const float* states, const float* actions, const float* returns, const float* advantages,
                              const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                              int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                         workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_train_step(const cpb_ppo_cat_spec* cspec, float* params, const float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                               int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_train_step(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, returns,
                          advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_train_step_opts(const cpb_ppo_cat_spec* cspec, float* params, const float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const float* returns,
                                    const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                    const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_train_step_opts(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                               returns, advantages, idx, batch, metrics, opts, stop, steps_applied, workspace,
                               workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads, float* adam_m,
                          float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                          const float* actions, const double* rewards, const double* values, double bootstrap_value,
                          const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                          int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, false, nullptr,
                     nullptr, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn_opts(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const double* rewards, const double* values,
                               double bootstrap_value, const double* dones, int32_t T, double gamma, double lam,
                               int32_t num_epochs, int32_t batch_size, const int32_t* perms, float* metrics,
                               const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, true, opts,
                     steps_applied, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn_segments(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                                   float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                   const float* states, const float* actions, const double* rewards,
                                   const double* values, const double* bootstrap_values, const double* dones,
                                   const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                   double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                   float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, false, nullptr, nullptr, workspace, workspace_bytes,
                              stream);
}

int32_t cpb_ppo_cat_learn_segments_opts(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                                        float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                        const float* states, const float* actions, const double* rewards,
                                        const double* values, const double* bootstrap_values, const double* dones,
                                        const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                        double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                        float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, true, opts, steps_applied, workspace,
                              workspace_bytes, stream);
}

// ---- The two-per-side entry points: the spec twins at {hidden1, hidden2} / {hidden1, hidden2}
#define CPB_PPO_SPEC_OF(cfg) \
    cpb_ppo_spec spec_;      \
    CPB_TRY(ppo_spec_of(cfg, &spec_));

int32_t cpb_ppo_layout(const cpb_ppo_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_layout(&spec_, offsets, sizes, shapes, total);
}

int64_t cpb_ppo_workspace_bytes(const cpb_ppo_config* cfg, int32_t max_batch, int32_t horizon) {
    cpb_ppo_spec spec_;
    if (ppo_spec_of(cfg, &spec_) != CPB_OK) return CPB_ERR_INVALID_ARGUMENT;
    return cpb_ppo_spec_workspace_bytes(&spec_, max_batch, horizon);
}

int32_t cpb_ppo_forward(const cpb_ppo_config* cfg, const float* params, const float* states, int32_t batch,
                        const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                        void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_forward(&spec_, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_loss_grad(const cpb_ppo_config* cfg, const float* params, const float* params_old,
                          const float* states, const float* actions, const float* returns, const float* advantages,
                          const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_loss_grad(&spec_, params, params_old, states, actions, returns, advantages, idx, batch, grads,
                                  metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_train_step(const cpb_ppo_config* cfg, float* params, const float* params_old, float* grads,
                           float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                           int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_train_step(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                                   returns, advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_train_step_opts(const cpb_ppo_config* cfg, float* params, const float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                const float* states, const float* actions, const float* returns,
                                const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_train_step_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                        actions, returns, advantages, idx, batch, metrics, opts, stop, steps_applied,
                                        workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                      float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                      const float* actions, const double* rewards, const double* values, double bootstrap_value,
                      const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                      int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                      int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics,
                              workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, double bootstrap_value,
                           const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                           int32_t batch_size, const int32_t* perms, float* metrics,
                           const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                                   rewards, values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms,
                                   metrics, opts, steps_applied, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn_segments(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                               float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const double* rewards, const double* values,
                               const double* bootstrap_values, const double* dones, const int32_t* segment_offsets,
                               int32_t num_segments, int32_t rows, double gamma, double lam, int32_t num_epochs,
                               int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_segments(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                       actions, rewards, values, bootstrap_values, dones, segment_offsets, num_segments,
                                       rows, gamma, lam, num_epochs, batch_size, perms, metrics, workspace,
                                       workspace_bytes, stream);
}

int32_t cpb_ppo_learn_segments_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                    double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                    float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_segments_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                            actions, rewards, values, bootstrap_values, dones, segment_offsets,
                                            num_segments, rows, gamma, lam, num_epochs, batch_size, perms, metrics, opts,
                                            steps_applied, workspace, workspace_bytes, stream);
}

}  // extern "C"
