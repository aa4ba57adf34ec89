/*
 * carla_ppo_b200.h -- C ABI of libcarla_ppo_b200.so: the H100 (sm_90a) implementation of the
 * neural hot path of bitsauce/Carla-ppo (ConvVAE train step + PPO update).
 *
 * The reference has no FFI: its boundary is the Python class surface of vae/models.py, ppo.py and
 * utils.py over `tf.Session.run` (SURVEY.md section 8b).  This header is what a maintainer would
 * bind (ctypes, see INTEGRATION.md) to replace each `sess.run` on that path; every entry point
 * cites the reference call it replaces (paths relative to the reference repo root).
 *
 * Conventions
 *   - plain pointers and sizes only.  Unless the name ends in `_host`, every data pointer is a
 *     DEVICE pointer (cudaMalloc'd by the caller, e.g. a torch tensor's data_ptr()); tensors are
 *     dense, row-major, NHWC for images, exactly the layouts of the reference's placeholders and
 *     TF variables.  `stream` is a cudaStream_t passed as void*; all work is enqueued on it and no
 *     entry point synchronises unless documented.
 *   - model state (parameters, gradients, Adam m/v) lives in FLAT float32 buffers owned by the
 *     caller; cpb_vae_layout / cpb_ppo_layout give each TF variable's offset in that buffer.
 *   - every function returns 0 on success or a negative cpb_status; cpb_last_error() returns a
 *     message for the calling thread.  Bad arguments never launch anything.
 *   - geometry: source frames are [B,H,W,3], targets [B,H,W,Ct] with Ct in {3,1}.  The ConvVAE takes
 *     any H and W that are multiples of 16 in [48,512] through the cpb_vae_spec_* entry points (the
 *     frame sizes the reference's ConvVAE builds, vae/models.py:233-268); the cpb_vae_config entry
 *     points and the MlpVAE use the reference's default 80x160 (vae_common.py:18-20).  z_dim must be a
 *     multiple of 4 in [4,1024] (ConvVAE and MlpVAE).  Every [B,z] latent row (eps, mean, logvar, z,
 *     latent) is dense at pitch z_dim.
 */
#ifndef CARLA_PPO_B200_H
#define CARLA_PPO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    CPB_OK = 0,
    CPB_ERR_INVALID_ARGUMENT = -1,
    CPB_ERR_CUDA = -2,
    CPB_ERR_WORKSPACE_TOO_SMALL = -3,
    CPB_ERR_UNSUPPORTED = -4
} cpb_status;

/* loss selectors: vae/models.py:11-22 (bce_loss, bce_loss_v2, mse_loss) */
enum { CPB_LOSS_MSE = 0, CPB_LOSS_BCE = 1, CPB_LOSS_BCE_V2 = 2 };
/* frame element types accepted for source / target images */
enum { CPB_FRAME_F32 = 0, CPB_FRAME_U8 = 1 };
/* workspace sizing modes */
enum { CPB_WS_ENCODE = 0, CPB_WS_FORWARD = 1, CPB_WS_TRAIN = 2 };

const char* cpb_last_error(void);
/* "sm_90a" build tag + version, for diagnostics */
const char* cpb_build_info(void);

/* ------------------------------------------------------------------------------------------
 * ConvVAE (vae/models.py:233-268 on top of VAE.__init__ :38-159)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t batch;            /* frames in this call (per rank) */
    int32_t target_channels;  /* 3 = rgb target, 1 = segmentation target (vae_common.py:15) */
    int32_t z_dim;            /* latent size: a multiple of 4 in [4,1024] (64 in every shipped model) */
    int32_t loss_type;        /* CPB_LOSS_* */
    int32_t source_dtype;     /* CPB_FRAME_F32: values in [0,1]; CPB_FRAME_U8: raw 0..255, scaled by 1/255 */
    int32_t target_dtype;     /* CPB_FRAME_F32, or CPB_FRAME_U8 scaled by target_u8_scale */
    float   target_u8_scale;  /* 1/255 for rgb, 1/12 for class ids (vae/train_vae.py:15-29) */
    float   beta;             /* KL weight (vae/models.py:137) */
    float   kl_tolerance;     /* vae/models.py:133-134 */
    float   loss_scale;       /* multiplies both batch means and all gradients: 1 for a whole batch,
                                 shard/global for a data-parallel shard (sum over ranks = global mean) */
} cpb_vae_config;

/* A ConvVAE at any legal frame size: H = height and W = width, each a multiple of 16 in [48, 512].  The encoder's
 * four 4x4 stride-2 VALID convolutions give H1 = H/2 - 1, H2 = H/4 - 2, H3 = H/8 - 2, H4 = H/16 - 2 (the same in W) and
 * FEAT = H4*W4*256; the decoder maps H4 back to exactly H (any other height fails the reference's assert,
 * vae/models.py:265).  The variables keep their names, TF shapes and storage order; only mean, logstd_sqare and
 * dense1 grow with FEAT.  Every cpb_vae_* entry point below has a cpb_vae_spec_* twin with the same arguments, the spec
 * in place of the config; the cpb_vae_* ones are the twins at {cfg, 80, 160}.  A frame outside the rule is refused
 * (CPB_ERR_INVALID_ARGUMENT) before any launch.
 * Batch bound: in math modes 1 and 2 the tensor-core kernels address a tensor with 32-bit offsets, which needs
 * B * H1 * W1 * 32 < 2^31 (B <= 21781 at 80x160, 5342 at 160x320, 1032 at 512x512); a larger batch is refused with
 * CPB_ERR_UNSUPPORTED before any launch.  Math mode 0 takes every batch. */
typedef struct {
    cpb_vae_config base;      /* batch, target_channels, z_dim, loss, dtypes, beta, kl_tolerance, loss_scale */
    int32_t height, width;    /* H, W of the source and target frames */
} cpb_vae_spec;

/* Number of TF variables (22) and their names, in creation order ("encoder/conv1/kernel", ...,
 * without the leading "vae/" scope).  Replaces: tf.trainable_variables() of the "vae" scope. */
int32_t     cpb_vae_num_tensors(void);
const char* cpb_vae_tensor_name(int32_t index);
/* Offsets/sizes (in floats) of every variable inside the flat parameter buffer and its total length
 * (offsets are 64-float aligned; padding floats must be zero).  shapes: 4 ints per tensor, TF shape
 * padded with 0.  Any output pointer may be NULL. */
int32_t cpb_vae_layout(int32_t target_channels, int32_t z_dim, int64_t* offsets, int64_t* sizes,
                       int32_t* shapes, int64_t* total_floats);
/* Bytes of scratch the calls below need for `batch` frames (mode = CPB_WS_*). */
int64_t cpb_vae_workspace_bytes(int32_t batch, int32_t target_channels, int32_t z_dim, int32_t mode);

/* VAE.encode (vae/models.py:199-202): mean[B,z]; logvar[B,z] optional (NULL to skip).
 * flags (optional int32[1]): bit0 set when a source value is outside [0,1] (verify_range, :24-30). */
int32_t cpb_vae_encode(const cpb_vae_config* cfg, const float* params, const void* source,
                       float* mean, float* logvar, int32_t* flags,
                       void* workspace, int64_t workspace_bytes, void* stream);

/* VAE.generate_from_latent (vae/models.py:188-191): sigmoid(decoder(z)) flattened [B, 80*160*Ct]. */
int32_t cpb_vae_decode(const cpb_vae_config* cfg, const float* params, const float* z,
                       float* reconstruction, void* workspace, int64_t workspace_bytes, void* stream);

/* The training graph without the optimiser (VAE.evaluate, vae/models.py:220-231):
 * losses[0] = reconstruction loss, losses[1] = KL loss (batch means x loss_scale).
 * eps[B,z] are the standard-normal draws of `normal.sample` (:103); eps == NULL means z = mean
 * (training=False, :105).  Optional outputs (NULL to skip): mean, logvar, z [B,z],
 * reconstruction = sigmoid(logits) [B, 80*160*Ct] (VAE.reconstruct, :193-197).
 * flags bit0: source out of [0,1]; bit1: target out of [0,1]. */
int32_t cpb_vae_forward(const cpb_vae_config* cfg, const float* params, const void* source,
                        const void* target, const float* eps, float* losses,
                        float* mean, float* logvar, float* z, float* reconstruction, int32_t* flags,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* Forward + reverse-mode gradient of (recon + beta*kl) w.r.t. all 22 variables, written into the
 * flat `grads` buffer (same layout as params; fully overwritten).  Replaces the tf.gradients half
 * of optimizer.minimize (vae/models.py:141-142).  Between this call and cpb_adam_apply a
 * data-parallel caller all-reduces (sum) `grads` and `losses`. */
int32_t cpb_vae_loss_grad(const cpb_vae_config* cfg, const float* params, const void* source,
                          const void* target, const float* eps, float* grads, float* losses,
                          int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);

/* TF-1.13 ApplyAdam on a flat buffer (22 x ApplyAdam in the VAE graph, 13 in the PPO graph):
 *   alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)
 *   m += (g - m)(1 - beta1);  v += (g*g - v)(1 - beta2);  p -= alpha * m / (sqrt(v) + eps)
 * then powers[0] *= beta1, powers[1] *= beta2 (device float[2], initialised to {beta1, beta2}).
 * lr_dev (optional device float[1]) overrides `lr` when non-NULL (PPO's decayed rate). */
int32_t cpb_adam_apply(float* params, const float* grads, float* m, float* v, int64_t n,
                       float* powers, float lr, const float* lr_dev, float beta1, float beta2,
                       float epsilon, void* stream);

/* The same with a guard: `guard` (nullable) points at one 32-bit device word; when any of its bits is set the whole
 * update (parameters, m, v, beta powers) is skipped.  Used with the verify_range flag word: the reference's tf.Assert
 * (vae/models.py:24-30) aborts the sess.run before ApplyAdam, so an out-of-range batch must not touch the model.
 * A data-parallel caller passes the all-reduced flag (any 32-bit pattern, e.g. a float sum; only == 0 matters). */
int32_t cpb_adam_apply_guarded(float* params, const float* grads, float* m, float* v, int64_t n,
                               float* powers, float lr, const float* lr_dev, float beta1, float beta2,
                               float epsilon, const void* guard, void* stream);

/* One reference minibatch step: sess.run([train_step, ...]) of VAE.train_one_epoch
 * (vae/models.py:213-216) = cpb_vae_loss_grad + cpb_adam_apply_guarded(guard = flags) on one GPU: when `flags` is given
 * and a source/target value is outside [0,1], the losses are still written but the model is left untouched. */
int32_t cpb_vae_train_step(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, float lr, const void* source,
                           const void* target, const float* eps, float* losses, int32_t* flags,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* Same step fed like the reference feeds it: source/target/eps are HOST buffers (numpy arrays of the
 * feed_dict).  Copies them into `staging` (device, cpb_vae_staging_bytes), runs the step, copies
 * losses[2] and flags back to the host pointers and synchronises the stream.  target_host may equal
 * source_host (rgb target): it is then uploaded once. */
int64_t cpb_vae_staging_bytes(const cpb_vae_config* cfg);
int32_t cpb_vae_train_step_host(const cpb_vae_config* cfg, float* params, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, float lr, const void* source_host,
                                const void* target_host, const float* eps_host, float* losses_host,
                                int32_t* flags_host, void* staging, int64_t staging_bytes,
                                void* workspace, int64_t workspace_bytes, void* stream);

/* The cpb_vae_spec twins.  layout reads target_channels, z_dim, height and width; workspace_bytes also the batch. */
int32_t cpb_vae_spec_layout(const cpb_vae_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                            int64_t* total_floats);
int64_t cpb_vae_spec_workspace_bytes(const cpb_vae_spec* spec, int32_t mode);
int32_t cpb_vae_spec_encode(const cpb_vae_spec* spec, const float* params, const void* source,
                            float* mean, float* logvar, int32_t* flags,
                            void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_vae_spec_decode(const cpb_vae_spec* spec, const float* params, const float* z,
                            float* reconstruction, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_vae_spec_forward(const cpb_vae_spec* spec, const float* params, const void* source,
                             const void* target, const float* eps, float* losses,
                             float* mean, float* logvar, float* z, float* reconstruction, int32_t* flags,
                             void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_vae_spec_loss_grad(const cpb_vae_spec* spec, const float* params, const void* source,
                               const void* target, const float* eps, float* grads, float* losses,
                               int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_vae_spec_train_step(const cpb_vae_spec* spec, float* params, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, float lr, const void* source,
                                const void* target, const float* eps, float* losses, int32_t* flags,
                                void* workspace, int64_t workspace_bytes, void* stream);
int64_t cpb_vae_spec_staging_bytes(const cpb_vae_spec* spec);
int32_t cpb_vae_spec_train_step_host(const cpb_vae_spec* spec, float* params, float* grads, float* adam_m,
                                     float* adam_v, float* adam_powers, float lr, const void* source_host,
                                     const void* target_host, const float* eps_host, float* losses_host,
                                     int32_t* flags_host, void* staging, int64_t staging_bytes,
                                     void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * MlpVAE (vae/models.py:271-299): flatten(38400) -> one dense relu layer per encoder size -> mean / logstd_sqare heads ->
 * sample -> one dense relu layer per decoder size -> the output layer, dense 12800*Ct (logits).  Same conventions as the
 * ConvVAE entry points above (flat parameter buffer described by the layout call, caller-owned workspace, same loss /
 * flag semantics); the optimiser is cpb_adam_apply(_guarded) on the flat buffers.
 * Shapes: 1 to 8 hidden layers per side, every width a multiple of 32 in [32, 8192] (an empty side is refused).
 * Variables, in the reference's creation order (build_mlp, vae/models.py:283-296), each {kernel [in,out], bias}:
 * encoder/dense, encoder/dense_1 ... encoder/dense_{L-1}, mean, logstd_sqare, decoder/dense ... decoder/dense_{M-1} and
 * the output layer decoder/dense_M [dec_{M-1}, 12800*Ct]: 2 (L + M + 3) tensors.
 * Arithmetic: fp32 SIMT in math modes 0 and 1.  In math mode 2 (cpb_set_math_mode) the five frame-wide products -- the
 * first encoder layer's forward and weight gradient, the output layer's forward, data gradient and weight gradient --
 * run as ONE TF32 wgmma pass with both operands rounded to nearest; everything else (the other hidden layers, the heads,
 * sampling, loss, Adam) runs as in the other modes.
 * Batches with batch * 38400 >= 2^31 run those five products on the fp32 kernels in every mode.
 * The workspace size depends on the math mode at the time of the query: mode 2 adds the TF32 weight images and the
 * split partials, and a mode-2 call given a smaller workspace fails with CPB_ERR_WORKSPACE_TOO_SMALL.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    cpb_vae_config base;               /* batch, target_channels, z_dim, loss, dtypes, beta, kl_tolerance, loss_scale */
    int32_t num_encoder;               /* L = len(encoder_sizes), 1..8 */
    int32_t encoder_sizes[8];          /* the first L are used */
    int32_t num_decoder;               /* M = len(decoder_sizes), 1..8 */
    int32_t decoder_sizes[8];          /* the first M are used */
} cpb_mlpvae_spec;

int32_t     cpb_mlpvae_spec_num_tensors(const cpb_mlpvae_spec* spec);          /* 2 (L + M + 3) */
const char* cpb_mlpvae_spec_tensor_name(const cpb_mlpvae_spec* spec, int32_t index);
int32_t cpb_mlpvae_spec_layout(const cpb_mlpvae_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes /* 4 per tensor */,
                               int64_t* total_floats);
int64_t cpb_mlpvae_spec_workspace_bytes(const cpb_mlpvae_spec* spec, int32_t mode);
int32_t cpb_mlpvae_spec_encode(const cpb_mlpvae_spec* spec, const float* params, const void* source, float* mean, float* logvar,
                               int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_spec_decode(const cpb_mlpvae_spec* spec, const float* params, const float* z, float* reconstruction,
                               void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_spec_forward(const cpb_mlpvae_spec* spec, const float* params, const void* source, const void* target,
                                const float* eps, float* losses, float* mean, float* logvar, float* z, float* reconstruction,
                                int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_spec_loss_grad(const cpb_mlpvae_spec* spec, const float* params, const void* source, const void* target,
                                  const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                                  int64_t workspace_bytes, void* stream);

/* The reference's default shape, two hidden layers per side: the cpb_mlpvae_spec_* entry points on
 * {enc1, enc2} / {dec1, dec2}, with the same meaning and results. */
typedef struct {
    cpb_vae_config base;               /* batch, target_channels, z_dim, loss, dtypes, beta, kl_tolerance, loss_scale */
    int32_t enc1, enc2;                /* encoder_sizes (512, 256)   (vae/models.py:277) */
    int32_t dec1, dec2;                /* decoder_sizes (256, 512)   (vae/models.py:278) */
} cpb_mlpvae_config;

int32_t     cpb_mlpvae_num_tensors(void);              /* 14 */
const char* cpb_mlpvae_tensor_name(int32_t index);
int32_t cpb_mlpvae_layout(const cpb_mlpvae_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes /* 4 per tensor */,
                          int64_t* total_floats);
int64_t cpb_mlpvae_workspace_bytes(const cpb_mlpvae_config* cfg, int32_t mode);
int32_t cpb_mlpvae_encode(const cpb_mlpvae_config* cfg, const float* params, const void* source, float* mean, float* logvar,
                          int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_decode(const cpb_mlpvae_config* cfg, const float* params, const float* z, float* reconstruction,
                          void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_forward(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target,
                           const float* eps, float* losses, float* mean, float* logvar, float* z, float* reconstruction,
                           int32_t* flags, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_mlpvae_loss_grad(const cpb_mlpvae_config* cfg, const float* params, const void* source, const void* target,
                             const float* eps, float* grads, float* losses, int32_t* flags, void* workspace,
                             int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * PPO (ppo.py, utils.py:45-50, train.py:171-207)
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t state_dim;        /* 67 = 64-d latent + steer, throttle, speed (train.py:68,85) */
    int32_t num_actions;      /* 2 */
    int32_t hidden1, hidden2; /* 500, 300 for both trunks (ppo.py:17); 0 in a cpb_ppo_spec */
    float   action_low[4];    /* action_space.low / .high (ppo.py:38) */
    float   action_high[4];
    float   epsilon;          /* clip range (ppo.py:124) */
    float   value_scale;      /* ppo.py:127 */
    float   entropy_scale;    /* ppo.py:130 */
} cpb_ppo_config;

/* The policy and value networks with their own lists of hidden-layer sizes (Stable-Baselines3's
 * net_arch=dict(pi=[...], vf=[...])): num_policy / num_value dense + ReLU layers (1..8 each, every width >= 1) from the
 * state to the action head and to the value head.  base.hidden1 / base.hidden2 must be 0 (refused otherwise: the widths
 * are the lists).  Variables, in TF creation order and naming (ppo.py:38-66), 2P + 2V + 5 of them:
 *   dense, dense_1 .. dense_{P-1} (kernel, bias), action_mean/kernel, action_mean/bias, action_logstd,
 *   dense_P .. dense_{P+V-1} (kernel, bias), value/kernel, value/bias.
 * Every cpb_ppo_* entry point below on a cpb_ppo_config is its cpb_ppo_spec_* twin at {hidden1, hidden2} /
 * {hidden1, hidden2}: same layout, workspace, launches and results.  A bad spec (NULL, a depth outside [1, 8], a width
 * < 1, nonzero base.hidden*, num_actions outside [1, 4]) is refused with CPB_ERR_INVALID_ARGUMENT before anything is
 * enqueued.  Under CPB_PPO_PERSISTENT=1 the learn twins run every architecture in the persistent kernel. */
#define CPB_PPO_MAX_LAYERS 8
typedef struct {
    cpb_ppo_config base;      /* hidden1 = hidden2 = 0 */
    int32_t num_policy;
    int32_t policy_sizes[CPB_PPO_MAX_LAYERS];
    int32_t num_value;
    int32_t value_sizes[CPB_PPO_MAX_LAYERS];
} cpb_ppo_spec;

int32_t     cpb_ppo_num_tensors(void);             /* 13 */
const char* cpb_ppo_tensor_name(int32_t index);    /* "dense/kernel", ... (scope-relative) */
int32_t cpb_ppo_layout(const cpb_ppo_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                       int64_t* total_floats);
int64_t cpb_ppo_workspace_bytes(const cpb_ppo_config* cfg, int32_t max_batch, int32_t horizon);

/* PPO.predict (ppo.py:231-251) without the sampling: action_mean[B,A], value[B].
 * noise (optional [B,A] standard-normal): action = clip(mean + noise*exp(logstd), low, high). */
int32_t cpb_ppo_forward(const cpb_ppo_config* cfg, const float* params, const float* states,
                        int32_t batch, const float* noise, float* action, float* value,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* Loss + gradient of one minibatch (ppo.py:119-144, without ApplyAdam).
 * metrics[5] = policy_loss, value_loss, entropy_loss, loss, mean(prob_ratio).
 * idx (optional int32[batch]): gather rows idx[i] of states/actions/returns/advantages first
 * (the reference's states[mb_idx] fancy-index, train.py:204-207). */
int32_t cpb_ppo_loss_grad(const cpb_ppo_config* cfg, const float* params, const float* params_old,
                          const float* states, const float* actions, const float* returns,
                          const float* advantages, const int32_t* idx, int32_t batch,
                          float* grads, float* metrics, void* workspace, int64_t workspace_bytes,
                          void* stream);

/* PPO.train (ppo.py:218-229): cpb_ppo_loss_grad + ApplyAdam with lr_dev[0]. */
int32_t cpb_ppo_train_step(const cpb_ppo_config* cfg, float* params, const float* params_old,
                           float* grads, float* adam_m, float* adam_v, float* adam_powers,
                           const float* lr_dev, const float* states, const float* actions,
                           const float* returns, const float* advantages, const int32_t* idx,
                           int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes,
                           void* stream);

/* utils.compute_gae (utils.py:45-50) + train.py:176-177, float64 like the reference:
 *   delta_t = r_t + (1-d_t) gamma V_{t+1} - V_t ;  A_t = delta_t + gamma*lam*A_{t+1}  (no reset)
 *   returns = A + V ;  advantages_norm = (A - mean A) / (std A + 1e-8)
 * rewards, values, dones: double[T] (dones as 0/1); outputs double[T]: advantages is required,
 * returns and advantages_norm may be NULL. */
int32_t cpb_gae(const double* rewards, const double* values, double bootstrap_value,
                const double* dones, int32_t T, double gamma, double lam,
                double* advantages, double* returns, double* advantages_norm, void* stream);

/* The driver's whole update block (train.py:171-207) with no host round trip:
 * GAE -> returns -> normalised advantages -> theta_old <- theta -> num_epochs x ceil(T/batch)
 * minibatch Adam steps following perms[num_epochs][T] (int32 index order of each epoch; may be NULL when
 * num_epochs == 0).
 * metrics: float[num_epochs*ceil(T/batch)][5] (optional). */
int32_t cpb_ppo_learn(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                      float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                      const float* states, const float* actions, const double* rewards,
                      const double* values, double bootstrap_value, const double* dones, int32_t T,
                      double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                      const int32_t* perms, float* metrics, void* workspace,
                      int64_t workspace_bytes, void* stream);

/* One environment step of the reference's RL loop in ONE call with no host round trip in between (train.py:143 +
 * vae_common.py:45-61 + ppo.py:231-251): frames [B,80,160,3] (uint8 or fp32, per vae_cfg->source_dtype) -> VAE mean ->
 * state[b] = [latent(z) | measurements(M)] -> policy / value networks -> action (sampled with `noise`, or the mean when
 * noise == NULL) and value.  latent_tmp: scratch [B,z]; state [B,z+M], action [B,A], value [B] are outputs. */
int32_t cpb_encode_predict(const cpb_vae_config* vae_cfg, const float* vae_params, const void* frames,
                           const float* measurements, int32_t num_measurements,
                           const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                           float* latent_tmp, float* state, float* action, float* value, int32_t* flags,
                           void* vae_workspace, int64_t vae_workspace_bytes,
                           void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);

/* cpb_encode_predict with a ConvVAE at any legal frame size: frames [B,H,W,3] (spec->height, spec->width). */
int32_t cpb_vae_spec_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                    const float* measurements, int32_t num_measurements,
                                    const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                    float* latent_tmp, float* state, float* action, float* value, int32_t* flags,
                                    void* vae_workspace, int64_t vae_workspace_bytes,
                                    void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);

/* cpb_encode_predict with an MlpVAE (cpb_mlpvae_spec) as the encoder; same arguments, outputs and noise use. */
int32_t cpb_mlpvae_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                  const float* measurements, int32_t num_measurements,
                                  const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                  float* latent_tmp, float* state, float* action, float* value, int32_t* flags,
                                  void* vae_workspace, int64_t vae_workspace_bytes,
                                  void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);

/* Arithmetic used for the dense conv / transposed-conv contractions of the VAE (modes 1 and 0 are fp32-accurate):
 *   1 (default) wgmma tf32 with the error-compensated 3xTF32 split, fp32 accumulators in registers;
 *   0           fp32 FMA (SIMT) tap-GEMM -- also used in modes 1 and 2 for the layers the tensor-core kernel does
 *               not cover (3-channel edge layers, dense heads, weight gradients);
 *   2           ONE wgmma tf32 pass, NOT fp32-accurate: both operands are rounded to the nearest TF32 value (10-bit
 *               mantissa, ties away from zero), so each product carries a relative error of up to 2^-10 with no
 *               systematic sign; accumulation stays fp32 (chunks of 128 k added into fp32 registers).
 *               The comparable setting of cuDNN / TensorFlow on this hardware is their TF32 default.
 * Modes 1 and 2 cover the same layers of the ConvVAE: forward, data gradient and weight gradient of conv2-4 and
 * deconv1-3, in every entry point that runs them (encode, decode, forward, loss_grad, train_step(_host),
 * cpb_encode_predict).  conv1, deconv4, the heads, dense1, the dense weight gradients and PPO use the fp32 kernels
 * in every mode.  The MlpVAE uses the fp32 kernels in modes 0 and 1; mode 2 also runs its five frame-wide products
 * (first encoder layer forward + weight gradient, output layer forward + data gradient + weight gradient) as one TF32
 * pass (see the MlpVAE section).  The mode is process-global and read when a call is enqueued (and by the MlpVAE
 * workspace query); other values are rejected (CPB_ERR_INVALID_ARGUMENT). */
int32_t cpb_set_math_mode(int32_t mode);
/* Debug / test hooks (not part of the reference-facing surface): workspace buffer offsets in bytes for
 * [xp,a1,a2,a3,a4,heads,z,d1,b1,b2,b3,logits_p,gA,gB,frame_loss,kl_rows,gz,gheads] (-1 = absent in that mode; the
 * first min(18, capacity) entries are written and their count returned; new entries are only ever appended), and a
 * dense D[M,N] = A[M,K] * Bt[N,K]^T through the tensor-core kernel (scratch: at least 2*N*K floats, the weight image). */
int32_t cpb_debug_vae_buffer_offsets(int32_t batch, int32_t target_channels, int32_t z_dim, int32_t mode,
                                     int64_t* offsets, int32_t capacity);
/* The same for a ConvVAE at the spec's frame size (batch, target_channels, z_dim, height, width). */
int32_t cpb_debug_vae_spec_buffer_offsets(const cpb_vae_spec* spec, int32_t mode, int64_t* offsets, int32_t capacity);
/* Process-global, like the math mode: every later ConvVAE backward pass (loss_grad, train_step) returns CPB_OK right
 * after the named layer group -- its weight, bias and data gradients -- has been enqueued.  Groups in pass order:
 * "deconv4.dgrad", "deconv3.dgrad", "deconv2.dgrad", "deconv1.dgrad", "dense1.dgrad", "heads.dgrad", "conv4.dgrad",
 * "conv3.dgrad" (the whole pass ends with conv2's data gradient and conv1's weight gradient).  At a stop, the
 * workspace gradient buffer the group read (logits_p, gA, gB, gz or gheads) still holds its input gradient and the one
 * it wrote its output gradient; gradients of the layers not reached yet are 0.  NULL runs the whole pass again; any
 * other string is rejected (CPB_ERR_INVALID_ARGUMENT) and leaves the setting as it was. */
int32_t cpb_debug_vae_backward_stop(const char* group);
/* The MlpVAE twin, in the current math mode: [x,h_0..h_{L-1},heads,z,g_0..g_{M-1},logits,ga,gb], L + M + 6 entries
 * (ga / gb: the backward pass's two gradient buffers; after loss_grad, gb holds d loss / d (encoder/dense pre-activation)
 * and logits d loss / d logits).  The two-per-side call returns [x,h1,h2,heads,z,g1,g2,logits,ga,gb]. */
int32_t cpb_debug_mlpvae_spec_buffer_offsets(const cpb_mlpvae_spec* spec, int32_t mode, int64_t* offsets, int32_t capacity);
int32_t cpb_debug_mlpvae_buffer_offsets(const cpb_mlpvae_config* cfg, int32_t mode, int64_t* offsets, int32_t capacity);
int32_t cpb_debug_tc_wgrad(const float* big, const float* small, float* out, int32_t m, int32_t i, int32_t j,
                           int32_t variant, float* partial, void* stream);
int32_t cpb_debug_tc_gemm(const float* a, const float* bt, float* d, int32_t m, int32_t n, int32_t k,
                          float* scratch, void* stream);
int32_t cpb_get_math_mode(void);

/* Counters for bench.py's `gpu_launches`: kernels launched by this library since the last reset. */
int64_t cpb_launch_count(void);
void    cpb_reset_launch_count(void);

/* Optional per-call-site device timing (CUDA events recorded on the launching stream around each
 * labelled kernel group, e.g. "conv2.fwd", "deconv3.wgrad").  Off by default; bench.py turns it on for a
 * few extra steps AFTER the timed region to attribute the step time and compute the roofline figures.
 * cpb_profile_report synchronises the device and writes lines "label count total_ms\n" into buf. */
void    cpb_profile_enable(int32_t on);
void    cpb_profile_reset(void);
int64_t cpb_profile_report(char* buf, int64_t capacity);

/* ------------------------------------------------------------------------------------------
 * PPO over several trajectory segments (N environments stepped in lockstep)
 *
 * A segment is the contiguous run of rows [segment_offsets[s], segment_offsets[s+1]) that one environment produced
 * between two updates; segment_offsets[S+1] (int32, device) runs from 0 to rows and increases strictly, and its contents
 * are trusted like perms.  Within a segment the GAE is utils.compute_gae on that rollout (utils.py:45-50,
 * train.py:171-177): delta masks the bootstrap term by (1 - d), the accumulation is not reset inside the segment, and
 * bootstrap_values[s] follows its last row.  Returns are A + V per row; the advantages are normalised ONCE over all rows
 * (population std + 1e-8).  With S = 1 the results are bit-identical to cpb_gae / cpb_ppo_learn.
 * S >= 1, rows >= S and the required pointers are checked before any launch (CPB_ERR_INVALID_ARGUMENT).
 * ---------------------------------------------------------------------------------------- */

/* cpb_gae over S segments (utils.py:45-50 + train.py:176-177 per segment, one normalisation): rewards, values, dones
 * double[rows], bootstrap_values double[S]; advantages double[rows] is required, returns / advantages_norm may be NULL. */
int32_t cpb_gae_segments(const double* rewards, const double* values, const double* bootstrap_values,
                         const double* dones, const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                         double gamma, double lam, double* advantages, double* returns, double* advantages_norm,
                         void* stream);

/* cpb_ppo_learn (train.py:171-207) over S segments: the segmented GAE above, then theta_old <- theta, one old-policy
 * log-prob pass over all rows and num_epochs x ceil(rows/batch) minibatch Adam steps following perms[num_epochs][rows]
 * (launch-per-kernel, or the persistent kernel under CPB_PPO_PERSISTENT=1, as in cpb_ppo_learn).
 * Workspace: cpb_ppo_workspace_bytes(cfg, min(batch_size, rows), rows). */
int32_t cpb_ppo_learn_segments(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                               const float* states, const float* actions, const double* rewards,
                               const double* values, const double* bootstrap_values, const double* dones,
                               const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                               double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                               const int32_t* perms, float* metrics, void* workspace,
                               int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Bounded PPO updates: global gradient-norm clipping and approximate-KL early stopping on the device
 *
 * Additions over the reference (which has neither): the *_opts twins below take the arguments of their originals plus
 * `opts` and `steps_applied` (and train_step a stop word), and write 7-wide metrics rows.  Options are per call; a NULL
 * `opts` or a 0 field turns that guard off, and a negative, NaN or infinite field is refused (CPB_ERR_INVALID_ARGUMENT)
 * before anything is enqueued.  With both guards off the parameters, theta_old, Adam m / v, beta powers and metric
 * columns 0-4 are bit-identical to the original entry point's.
 *
 *   max_grad_norm > 0 (torch.nn.utils.clip_grad_norm_): per minibatch n = sqrt(sum g^2) over the 13 policy/ tensors (the
 *     flat grads buffer; its zero padding adds nothing), c = max_grad_norm / (n + 1e-6), and when c < 1 every gradient is
 *     multiplied by c before ApplyAdam.  The sums have a fixed order: a repeated call is bit-identical.
 *   target_kl > 0 (Stable-Baselines3's estimator and rule): each minibatch computes, in its own forward pass and before its
 *     Adam step, approx_kl = mean_b((r_b - 1) - log r_b) with r_b = exp(logp - logp_old).  If approx_kl > 1.5 * target_kl,
 *     neither that minibatch's Adam step nor any later one of the call is applied: params, Adam m / v and the beta powers
 *     are left as they are (theta_old <- theta still happens at the start of learn).  Every learn call starts fresh.
 *
 *   metrics: float[num_epochs * ceil(rows / batch)][7] (optional): the five columns of the original, approx_kl, and the
 *     pre-clip gradient norm n.  The row of the minibatch that stopped the update is written; every later row is NaN.
 *   steps_applied (optional, device int32[1]): set to the number of Adam steps the call applied.
 *   After a stop, `grads` is unspecified: the later minibatches are still enqueued (the host cannot know of the stop) and
 *   computed, but they do not touch the model.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    float max_grad_norm;      /* 0 = off */
    float target_kl;          /* 0 = off */
} cpb_ppo_learn_options;

int32_t cpb_ppo_learn_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                           float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                           const float* states, const float* actions, const double* rewards,
                           const double* values, double bootstrap_value, const double* dones, int32_t T,
                           double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                           const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                           int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);

int32_t cpb_ppo_learn_segments_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                                    double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                    const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                                    int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);

/* One minibatch step of a bounded update (the reference's Python loop over PPO.train, with the guards above): metrics
 * float[7]; steps_applied (optional) is set to 1 when the step was applied, else 0.  stop (device uint32[1], optional)
 * is the update's stop word, owned by the caller: zero it before the update's first step; a step whose approx_kl
 * exceeds 1.5 * target_kl sets it, and every step is skipped (NaN metrics row) while it is non-zero, so a loop of these
 * calls stops exactly as cpb_ppo_learn_opts does, with no host sync.  stop == NULL: the stop lasts for this call only. */
int32_t cpb_ppo_train_step_opts(const cpb_ppo_config* cfg, float* params, const float* params_old,
                                float* grads, float* adam_m, float* adam_v, float* adam_powers,
                                const float* lr_dev, const float* states, const float* actions,
                                const float* returns, const float* advantages, const int32_t* idx,
                                int32_t batch, float* metrics, const cpb_ppo_learn_options* opts,
                                uint32_t* stop, int32_t* steps_applied, void* workspace,
                                int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Spec twins: the entry points above for a cpb_ppo_spec (arguments after the first are those of the original).
 * Layout arrays hold cpb_ppo_spec_num_tensors(spec) entries (shapes: 2 per tensor).
 * ---------------------------------------------------------------------------------------- */
int32_t     cpb_ppo_spec_num_tensors(const cpb_ppo_spec* spec);                 /* 2P + 2V + 5 */
const char* cpb_ppo_spec_tensor_name(const cpb_ppo_spec* spec, int32_t index);  /* NULL for a bad spec or index */
int32_t cpb_ppo_spec_layout(const cpb_ppo_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                            int64_t* total_floats);
int64_t cpb_ppo_spec_workspace_bytes(const cpb_ppo_spec* spec, int32_t max_batch, int32_t horizon);
int32_t cpb_ppo_spec_forward(const cpb_ppo_spec* spec, const float* params, const float* states, int32_t batch,
                             const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                             void* stream);
int32_t cpb_ppo_spec_loss_grad(const cpb_ppo_spec* spec, const float* params, const float* params_old,
                               const float* states, const float* actions, const float* returns,
                               const float* advantages, const int32_t* idx, int32_t batch, float* grads,
                               float* metrics, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_train_step(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                const float* states, const float* actions, const float* returns,
                                const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_train_step_opts(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                     float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                     const float* states, const float* actions, const float* returns,
                                     const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                     const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                     void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_learn(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, double bootstrap_value,
                           const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                           int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                           int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_learn_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                const float* states, const float* actions, const double* rewards,
                                const double* values, double bootstrap_value, const double* dones, int32_t T,
                                double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                                int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_learn_segments(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                                    double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                    const int32_t* perms, float* metrics, void* workspace,
                                    int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_spec_learn_segments_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                         float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                         const float* states, const float* actions, const double* rewards,
                                         const double* values, const double* bootstrap_values, const double* dones,
                                         const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                                         double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                         const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                                         int32_t* steps_applied, void* workspace, int64_t workspace_bytes,
                                         void* stream);
/* cpb_vae_spec_encode_predict / cpb_mlpvae_encode_predict with the PPO described by a cpb_ppo_spec (checked
 * before the VAE is enqueued). */
int32_t cpb_vae_spec_ppo_spec_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                             const float* measurements, int32_t num_measurements,
                                             const cpb_ppo_spec* ppo_spec, const float* ppo_params, const float* noise,
                                             float* latent_tmp, float* state, float* action, float* value,
                                             int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
                                             void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);
int32_t cpb_mlpvae_ppo_spec_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                           const float* measurements, int32_t num_measurements,
                                           const cpb_ppo_spec* ppo_spec, const float* ppo_params, const float* noise,
                                           float* latent_tmp, float* state, float* action, float* value,
                                           int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
                                           void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Categorical policies: discrete action spaces (Stable-Baselines3's Discrete(n) / MultiDiscrete(nvec)), an addition
 * over the reference, whose policy is always the tanh-squashed Gaussian (ppo.py:38-66).
 *
 * K = spec.base.num_actions components (1..4); component k has n_k = num_categories[k] categories (2..64), and
 * N = sum n_k <= 64.  spec.base.action_low / action_high must be all 0.  The head computes logits
 * z = h_P W + b (W = action_logits/kernel [H_P, N], b = action_logits/bias [N], columns grouped by component in order),
 * p_k = softmax(z_k) with the max subtracted, log p = z - m - log sum exp(z - m), and per row
 *   logp(a) = sum_k log p_k[a_k],   H = sum_k -sum_i p_ki log p_ki.
 * loss = -policy_loss + value_loss - entropy_scale * mean_b H (policy and value terms, clip and tie rule as above);
 * metrics keep their columns, entropy_loss = entropy_scale * mean H, and the guarded rows add approx_kl and the pre-clip
 * norm as above.
 * Variables, in TF creation order, 2P + 2V + 4 of them (no action_logstd):
 *   dense .. dense_{P-1}, action_logits/kernel, action_logits/bias, dense_P .. dense_{P+V-1}, value/kernel, value/bias.
 * Actions: the `actions` [T, K] buffers hold the taken indices as integer-valued floats; an index outside [0, n_k) is
 * clamped into it.  forward writes action [B, K] the same way: greedy (noise == NULL) the first largest logit of each
 * component; sampled, noise [B, K] uniforms in [0, 1) and the smallest i with u < cumsum_i p_k (fp32, index order), or the
 * last index with p > 0 when rounding leaves u above the last partial sum.
 * Each cpb_ppo_cat_* entry point is the cpb_ppo_spec_* entry point of the same name with the categorical head: the same
 * arguments after the spec, the same launches.  A bad spec (NULL, anything cpb_ppo_spec refuses, an n_k outside [2, 64],
 * N > 64, a nonzero action_low / action_high) is refused with CPB_ERR_INVALID_ARGUMENT before anything is enqueued.
 * ---------------------------------------------------------------------------------------- */
#define CPB_PPO_MAX_LOGITS 64
typedef struct {
    cpb_ppo_spec spec;            /* the trunks and hyper-parameters; spec.base.num_actions = K */
    int32_t num_categories[4];    /* n_k, the first K are used */
} cpb_ppo_cat_spec;

int32_t     cpb_ppo_cat_num_tensors(const cpb_ppo_cat_spec* spec);                 /* 2P + 2V + 4 */
const char* cpb_ppo_cat_tensor_name(const cpb_ppo_cat_spec* spec, int32_t index);  /* NULL for a bad spec or index */
int32_t cpb_ppo_cat_layout(const cpb_ppo_cat_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                           int64_t* total_floats);
int64_t cpb_ppo_cat_workspace_bytes(const cpb_ppo_cat_spec* spec, int32_t max_batch, int32_t horizon);
/* PPO.predict over a discrete space: action [B,K] (indices as floats), value [B]; noise [B,K] uniforms or NULL (greedy) */
int32_t cpb_ppo_cat_forward(const cpb_ppo_cat_spec* spec, const float* params, const float* states, int32_t batch,
                            const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                            void* stream);
/* cpb_ppo_spec_loss_grad / train_step / train_step_opts with the categorical head */
int32_t cpb_ppo_cat_loss_grad(const cpb_ppo_cat_spec* spec, const float* params, const float* params_old,
                              const float* states, const float* actions, const float* returns,
                              const float* advantages, const int32_t* idx, int32_t batch, float* grads,
                              float* metrics, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_cat_train_step(const cpb_ppo_cat_spec* spec, float* params, const float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                               const float* states, const float* actions, const float* returns,
                               const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                               void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_cat_train_step_opts(const cpb_ppo_cat_spec* spec, float* params, const float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const float* returns,
                                    const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                    const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                    void* workspace, int64_t workspace_bytes, void* stream);
/* cpb_ppo_spec_learn / learn_opts / learn_segments / learn_segments_opts with the categorical head (launch-per-kernel,
 * or the persistent kernel under CPB_PPO_PERSISTENT=1) */
int32_t cpb_ppo_cat_learn(const cpb_ppo_cat_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                          float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                          const float* actions, const double* rewards, const double* values, double bootstrap_value,
                          const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                          int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                          int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_cat_learn_opts(const cpb_ppo_cat_spec* spec, float* params, float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                               const float* states, const float* actions, const double* rewards,
                               const double* values, double bootstrap_value, const double* dones, int32_t T,
                               double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                               const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                               int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_cat_learn_segments(const cpb_ppo_cat_spec* spec, float* params, float* params_old, float* grads,
                                   float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                   const float* states, const float* actions, const double* rewards,
                                   const double* values, const double* bootstrap_values, const double* dones,
                                   const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                                   double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                   const int32_t* perms, float* metrics, void* workspace,
                                   int64_t workspace_bytes, void* stream);
int32_t cpb_ppo_cat_learn_segments_opts(const cpb_ppo_cat_spec* spec, float* params, float* params_old, float* grads,
                                        float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                        const float* states, const float* actions, const double* rewards,
                                        const double* values, const double* bootstrap_values, const double* dones,
                                        const int32_t* segment_offsets, int32_t num_segments, int32_t rows,
                                        double gamma, double lam, int32_t num_epochs, int32_t batch_size,
                                        const int32_t* perms, float* metrics, const cpb_ppo_learn_options* opts,
                                        int32_t* steps_applied, void* workspace, int64_t workspace_bytes,
                                        void* stream);
/* cpb_vae_spec_ppo_spec_encode_predict / cpb_mlpvae_ppo_spec_encode_predict with a categorical PPO: action [B,K] holds
 * the indices as floats, noise [B,K] uniforms (NULL: greedy). */
int32_t cpb_vae_spec_ppo_cat_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                            const float* measurements, int32_t num_measurements,
                                            const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params, const float* noise,
                                            float* latent_tmp, float* state, float* action, float* value,
                                            int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
                                            void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);
int32_t cpb_mlpvae_ppo_cat_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                          const float* measurements, int32_t num_measurements,
                                          const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params, const float* noise,
                                          float* latent_tmp, float* state, float* action, float* value,
                                          int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
                                          void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Running normalisation: Stable-Baselines3's VecNormalize (an addition; the reference feeds raw states and rewards).
 *
 * Statistics are RunningMeanStd(epsilon=1e-4): a device double[2*dim + 1] = [mean | var | count], initially 0, 1, 1e-4.
 * Updating them with a batch of n rows computes the batch mean and variance (ddof 0, two-pass) in float64 and merges
 * them with Chan's formula: delta = mu_b - mu, t = c + n, mu' = mu + delta*n/t,
 * var' = (var*c + var_b*n + delta^2*c*n/t)/t, c' = t.  Every sum has a fixed order that depends only on the shape, so
 * equal inputs give bit-identical statistics and outputs.
 *
 * cpb_obs_normalize: x [batch, dim] -> out [batch, dim].  With update != 0 the statistics are first updated with the
 * batch; every row is then normalised with the (updated) statistics, clip((x - mu) / sqrt(var + epsilon), +-clip), in
 * float64 rounded once to fp32.  With update == 0 the statistics are only read.
 *
 * cpb_reward_normalize: the reward path of VecNormalize for the environments env_ids [batch] (distinct, in any order) of
 * num_envs, with the return statistics ret_stats (dim 1) and the discounted returns `returns` [num_envs] (float64,
 * caller-owned, start at 0).  For each stepped environment, in this order: returns[e] = returns[e]*gamma + rewards[i];
 * the statistics are updated with the batch returns[env_ids]; out[i] = clip(rewards[i] / sqrt(var + epsilon), +-clip);
 * returns[e] = 0 where dones[i] != 0.  env_ids live on the device and are not checked: an id outside [0, num_envs) is
 * clamped into it.
 *
 * Refused with CPB_ERR_INVALID_ARGUMENT before anything is enqueued: a NULL pointer, dim < 1 (a reward config's dim must
 * be 1), a clip that is <= 0, NaN or infinite, an epsilon that is <= 0 or not finite, gamma outside [0, 1], batch < 1,
 * num_envs < 1.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t dim;        /* columns of the statistics (1 for the returns) */
    float clip;         /* clip_obs / clip_reward (SB3's default: 10) */
    double epsilon;     /* added to var under the square root (SB3's default: 1e-8) */
} cpb_running_norm;

/* stats [2*dim + 1] <- mean 0, var 1, count 1e-4 (one kernel on `stream`) */
int32_t cpb_running_norm_init(const cpb_running_norm* cfg, double* stats, void* stream);
int32_t cpb_obs_normalize(const cpb_running_norm* cfg, double* stats, const float* x, int32_t batch, int32_t update,
                          float* out, void* stream);
int32_t cpb_reward_normalize(const cpb_running_norm* cfg, double* ret_stats, double* returns, const int32_t* env_ids,
                             const float* rewards, const int32_t* dones, int32_t batch, int32_t num_envs, double gamma,
                             float* out, void* stream);

/* The normalisation of an actor call (the *_encode_predict_norm twins).  `state` then holds the normalised state, made
 * in the launch that assembles it (no extra launch); with rewards != NULL the reward path of cpb_reward_normalize runs
 * on the call's batch B (env_ids, rewards, dones and rewards_out are [B]), one launch more.  rewards == NULL: no
 * rewards this step, and the reward fields are not read. */
typedef struct {
    cpb_running_norm obs;       /* obs.dim must be the PPO's state_dim */
    double* obs_stats;          /* [2*state_dim + 1] */
    int32_t update;             /* 0: the observation statistics are only read (evaluation) */
    cpb_running_norm reward;    /* dim 1 */
    double* ret_stats;          /* [3] */
    double* returns;            /* [num_envs] */
    const int32_t* env_ids;     /* [B] */
    const float* rewards;       /* [B], or NULL */
    const int32_t* dones;       /* [B] */
    int32_t num_envs;
    double gamma;
    float* rewards_out;         /* [B] */
} cpb_actor_norm;

/* The four actor entry points above with running normalisation: the same arguments, then `norm`. */
int32_t cpb_vae_spec_ppo_spec_encode_predict_norm(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                                  const float* measurements, int32_t num_measurements,
                                                  const cpb_ppo_spec* ppo_spec, const float* ppo_params,
                                                  const float* noise, float* latent_tmp, float* state, float* action,
                                                  float* value, int32_t* flags, void* vae_workspace,
                                                  int64_t vae_workspace_bytes, void* ppo_workspace,
                                                  int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm);
int32_t cpb_mlpvae_ppo_spec_encode_predict_norm(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                                const float* measurements, int32_t num_measurements,
                                                const cpb_ppo_spec* ppo_spec, const float* ppo_params,
                                                const float* noise, float* latent_tmp, float* state, float* action,
                                                float* value, int32_t* flags, void* vae_workspace,
                                                int64_t vae_workspace_bytes, void* ppo_workspace,
                                                int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm);
int32_t cpb_vae_spec_ppo_cat_encode_predict_norm(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                                 const float* measurements, int32_t num_measurements,
                                                 const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params,
                                                 const float* noise, float* latent_tmp, float* state, float* action,
                                                 float* value, int32_t* flags, void* vae_workspace,
                                                 int64_t vae_workspace_bytes, void* ppo_workspace,
                                                 int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm);
int32_t cpb_mlpvae_ppo_cat_encode_predict_norm(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                               const float* measurements, int32_t num_measurements,
                                               const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params,
                                               const float* noise, float* latent_tmp, float* state, float* action,
                                               float* value, int32_t* flags, void* vae_workspace,
                                               int64_t vae_workspace_bytes, void* ppo_workspace,
                                               int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm);

#ifdef __cplusplus
}
#endif
#endif /* CARLA_PPO_B200_H */
