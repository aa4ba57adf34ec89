// The actor call of a PPO rollout behind the C ABI: encode the frames with either VAE (through its public encode entry
// point), assemble the state from the latent and the measurements, and run the PPO forward -- every *encode_predict* entry
// point.
#include "vae_shared.cuh"

using namespace cpb;

extern "C" {

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

// The encode_predict entry points: `encode` on the VAE described by `vae` (whose common part is `base`), then the state
// assembly and the PPO forward, with the Gaussian head of ppo_spec or (cat_spec != NULL) the categorical head of
// cat_spec.  The PPO spec is checked before anything is enqueued.  with_norm (the *_norm twins): `norm` is checked too,
// the state is assembled normalised (vecnorm.cu) and, when it carries rewards, the reward path runs after the forward.
static int32_t encode_predict(const cpb_vae_config* base, const void* vae, EncodeMeanFn encode, const float* vae_params,
                              const void* frames, const float* measurements, int32_t num_measurements, const cpb_ppo_spec* ppo_spec,
                              const cpb_ppo_cat_spec* cat_spec, const float* ppo_params, const float* noise, float* latent_tmp,
                              float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                              int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream,
                              bool with_norm = false, const cpb_actor_norm* norm = nullptr) {
    if (cat_spec != nullptr) ppo_spec = &cat_spec->spec;
    CPB_REQUIRE(base && ppo_spec && frames && latent_tmp && state && action && value, "encode_predict: NULL pointer");
    CPB_REQUIRE(num_measurements >= 0 && (num_measurements == 0 || measurements != nullptr), "encode_predict: bad measurements");
    const int B = base->batch;
    const int32_t ppo_tensors = cat_spec ? cpb_ppo_cat_num_tensors(cat_spec) : cpb_ppo_spec_num_tensors(ppo_spec);   // checks the spec
    if (ppo_tensors < 0) return ppo_tensors;
    CPB_REQUIRE(ppo_spec->base.state_dim == base->z_dim + num_measurements, "encode_predict: state_dim %d != z_dim %d + %d measurements",
                ppo_spec->base.state_dim, base->z_dim, num_measurements);
    if (with_norm) CPB_TRY(check_actor_norm(norm, ppo_spec->base.state_dim, B));
    CPB_TRY(encode(vae, vae_params, frames, latent_tmp, flags, vae_workspace, vae_workspace_bytes, stream));
    if (with_norm) {
        CPB_TRY(launch_actor_obs_norm(norm, latent_tmp, base->z_dim, measurements, num_measurements, B, state, (cudaStream_t)stream));
    } else {
        const int total = B * ppo_spec->base.state_dim;
        assemble_state_kernel<<<cdiv(total, 128), 128, 0, (cudaStream_t)stream>>>(latent_tmp, measurements, B, base->z_dim, num_measurements, state);
        CPB_LAUNCHED();
    }
    if (cat_spec != nullptr)
        CPB_TRY(cpb_ppo_cat_forward(cat_spec, ppo_params, state, B, noise, action, value, ppo_workspace, ppo_workspace_bytes, stream));
    else
        CPB_TRY(cpb_ppo_spec_forward(ppo_spec, ppo_params, state, B, noise, action, value, ppo_workspace, ppo_workspace_bytes, stream));
    return with_norm ? launch_actor_reward_norm(norm, B, (cudaStream_t)stream) : CPB_OK;
}

int32_t cpb_vae_spec_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
                                    int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                    float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                                    int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    cpb_ppo_spec ppo_spec;
    CPB_TRY(ppo_spec_of(ppo_cfg, &ppo_spec));
    return cpb_vae_spec_ppo_spec_encode_predict(spec, vae_params, frames, measurements, num_measurements, &ppo_spec, ppo_params,
                                                noise, latent_tmp, state, action, value, flags, vae_workspace,
                                                vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

static int32_t conv_encode_mean(const void* vae, const float* params, const void* frames, float* latent, int32_t* flags, void* ws,
                                int64_t ws_bytes, void* stream) {
    return cpb_vae_spec_encode((const cpb_vae_spec*)vae, params, frames, latent, nullptr, flags, ws, ws_bytes, stream);
}

int32_t cpb_vae_spec_ppo_spec_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                             const float* measurements, int32_t num_measurements, const cpb_ppo_spec* ppo_spec,
                                             const float* ppo_params, const float* noise, float* latent_tmp, float* state,
                                             float* action, float* value, int32_t* flags, void* vae_workspace,
                                             int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes,
                                             void* stream) {
    return encode_predict(spec ? &spec->base : nullptr, spec, conv_encode_mean, vae_params, frames, measurements, num_measurements,
                          ppo_spec, nullptr, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_vae_spec_ppo_cat_encode_predict(const cpb_vae_spec* spec, const float* vae_params, const void* frames,
                                            const float* measurements, int32_t num_measurements, const cpb_ppo_cat_spec* ppo_spec,
                                            const float* ppo_params, const float* noise, float* latent_tmp, float* state,
                                            float* action, float* value, int32_t* flags, void* vae_workspace,
                                            int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes,
                                            void* stream) {
    return encode_predict(spec ? &spec->base : nullptr, spec, conv_encode_mean, vae_params, frames, measurements, num_measurements,
                          nullptr, ppo_spec, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_vae_spec_ppo_spec_encode_predict_norm(const cpb_vae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
        int32_t num_measurements, const cpb_ppo_spec* ppo_spec, const float* ppo_params, const float* noise, float* latent_tmp,
        float* state, float* action, float* value, int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
        void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm) {
    return encode_predict(spec ? &spec->base : nullptr, spec, conv_encode_mean, vae_params, frames, measurements, num_measurements,
                          ppo_spec, nullptr, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream, true, norm);
}

int32_t cpb_vae_spec_ppo_cat_encode_predict_norm(const cpb_vae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
        int32_t num_measurements, const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params, const float* noise, float* latent_tmp,
        float* state, float* action, float* value, int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
        void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm) {
    return encode_predict(spec ? &spec->base : nullptr, spec, conv_encode_mean, vae_params, frames, measurements, num_measurements,
                          nullptr, ppo_spec, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream, true, norm);
}

int32_t cpb_encode_predict(const cpb_vae_config* vae_cfg, const float* vae_params, const void* frames, const float* measurements,
                           int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                           float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                           int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    return cpb_vae_spec_encode_predict(DefaultFrame(vae_cfg).p, vae_params, frames, measurements, num_measurements, ppo_cfg,
                                       ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                                       vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_mlpvae_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
                                  int32_t num_measurements, const cpb_ppo_config* ppo_cfg, const float* ppo_params, const float* noise,
                                  float* latent_tmp, float* state, float* action, float* value, int32_t* flags, void* vae_workspace,
                                  int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream) {
    cpb_ppo_spec ppo_spec;
    CPB_TRY(ppo_spec_of(ppo_cfg, &ppo_spec));
    return cpb_mlpvae_ppo_spec_encode_predict(spec, vae_params, frames, measurements, num_measurements, &ppo_spec, ppo_params, noise,
                                              latent_tmp, state, action, value, flags, vae_workspace, vae_workspace_bytes,
                                              ppo_workspace, ppo_workspace_bytes, stream);
}

static int32_t mlp_encode_mean(const void* vae, const float* params, const void* frames, float* latent, int32_t* flags, void* ws,
                               int64_t ws_bytes, void* stream) {
    return cpb_mlpvae_spec_encode((const cpb_mlpvae_spec*)vae, params, frames, latent, nullptr, flags, ws, ws_bytes, stream);
}

int32_t cpb_mlpvae_ppo_spec_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                           const float* measurements, int32_t num_measurements, const cpb_ppo_spec* ppo_spec,
                                           const float* ppo_params, const float* noise, float* latent_tmp, float* state,
                                           float* action, float* value, int32_t* flags, void* vae_workspace,
                                           int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes,
                                           void* stream) {
    return encode_predict(spec ? &spec->base : nullptr, spec, mlp_encode_mean, vae_params, frames, measurements, num_measurements,
                          ppo_spec, nullptr, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_mlpvae_ppo_cat_encode_predict(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames,
                                          const float* measurements, int32_t num_measurements, const cpb_ppo_cat_spec* ppo_spec,
                                          const float* ppo_params, const float* noise, float* latent_tmp, float* state,
                                          float* action, float* value, int32_t* flags, void* vae_workspace,
                                          int64_t vae_workspace_bytes, void* ppo_workspace, int64_t ppo_workspace_bytes,
                                          void* stream) {
    return encode_predict(spec ? &spec->base : nullptr, spec, mlp_encode_mean, vae_params, frames, measurements, num_measurements,
                          nullptr, ppo_spec, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream);
}

int32_t cpb_mlpvae_ppo_spec_encode_predict_norm(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
        int32_t num_measurements, const cpb_ppo_spec* ppo_spec, const float* ppo_params, const float* noise, float* latent_tmp,
        float* state, float* action, float* value, int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
        void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm) {
    return encode_predict(spec ? &spec->base : nullptr, spec, mlp_encode_mean, vae_params, frames, measurements, num_measurements,
                          ppo_spec, nullptr, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream, true, norm);
}

int32_t cpb_mlpvae_ppo_cat_encode_predict_norm(const cpb_mlpvae_spec* spec, const float* vae_params, const void* frames, const float* measurements,
        int32_t num_measurements, const cpb_ppo_cat_spec* ppo_spec, const float* ppo_params, const float* noise, float* latent_tmp,
        float* state, float* action, float* value, int32_t* flags, void* vae_workspace, int64_t vae_workspace_bytes,
        void* ppo_workspace, int64_t ppo_workspace_bytes, void* stream, const cpb_actor_norm* norm) {
    return encode_predict(spec ? &spec->base : nullptr, spec, mlp_encode_mean, vae_params, frames, measurements, num_measurements,
                          nullptr, ppo_spec, ppo_params, noise, latent_tmp, state, action, value, flags, vae_workspace,
                          vae_workspace_bytes, ppo_workspace, ppo_workspace_bytes, stream, true, norm);
}

}  // extern "C"
