// What the ConvVAE (conv_vae.cu), the MlpVAE (mlp_vae.cu) and the library runtime (runtime.cu) share: the math mode and
// the per-device setup, the configuration checks, the tap-GEMM's dense problem, the latent block of both VAEs and the
// workspace check.  The functions below vae_shared.cu defines are hidden: the library's dynamic symbols stay the C ABI.
#pragma once
#include "elementwise.cuh"
#include "tapgemm.cuh"
#include "wgrad.cuh"

namespace cpb {

extern int g_math_mode;     // cpb_set_math_mode: 0 fp32 SIMT, 1 3xTF32 wgmma, 2 single-pass TF32 wgmma (runtime.cu)
int32_t ensure_init();      // the per-device one-time kernel setup (runtime.cu)

#pragma GCC visibility push(hidden)

int tc_passes();            // the tensor-core kernels' passes in the current math mode: 3 (3xTF32) or 1 (runtime.cu)
int tc_debug_flags();       // CPB_TC_DEBUG (runtime.cu)

// The reference's frame, 80x160: the ConvVAE's cpb_vae_config entry points and the MlpVAE's input
constexpr int kDefaultH = 80, kDefaultW = 160;
// The cpb_vae_spec of a cpb_vae_config at 80x160 (a NULL cfg gives a NULL spec, which the spec entry points refuse)
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

// Inside the library the latent has z_pad = 64 * ceil(z / 64) columns: the heads and dense1 then run the shapes of a
// multiple-of-64 model (the k-split tap-GEMM needs N % 64 == 0).  The padded columns hold zeros.
int z_pad(int z);
// multiples of 4: every [B, z] row that crosses the ABI starts 16-byte aligned, so the pitch changes move float4
bool z_ok(int z);
#define CPB_Z_RULE "z_dim=%d must be a multiple of 4 in [4,1024]"
int32_t check_cfg(const cpb_vae_config* cfg);
// every VAE entry point, once its configuration is valid: the device is set up, the workspace given and `need` bytes large
int32_t check_workspace(const void* workspace, int64_t workspace_bytes, int64_t need);

TapGemmParams base_params();
// dense: dst[b, :N] = src[b, :K] @ W[K, ldw] (+bias)
TapGemmParams dense_problem(const float* src, int B, int K, const float* W, int N, const float* bias, const float* mask,
                            float* dst, int relu);
// out[k_real][j_real] = x[B, K]^T g[B, J], dropping the padded rows k >= k_real and columns j >= j_real
int32_t run_dense_wgrad(const char* label, const float* x, int K, int k_real, const float* g, int B, int J, int j_real,
                        float* partial, float* out, cudaStream_t s);
void add_relayout(RelayoutTable& t, int64_t src, int64_t dst, int taps, int rows, int cols, int mode, int rows_pad,
                  int cols_pad);

// The latent block both VAEs share: the two heads (mean, logstd_sq) over a [B, K] layer, z_pad-column latent rows
struct Latent {
    int B, K, z, zp;
    const int64_t* off;     // the VAE's parameter offsets
    int mean;               // tensor index of mean/kernel; mean/bias, logstd_sqare/kernel and logstd_sqare/bias follow it
};

// Both heads as one y-batched dense problem over x [B, K]: heads[0] = mean, heads[1] = logstd_sq.  The weights are the
// parameters (both kernels, and both biases, are adjacent) when z == z_pad, the zero-padded wp and bp otherwise.
TapGemmParams heads_fwd_problem(const Latent& h, const float* params, const float* x, const float* wp, const float* bp,
                                float* heads);
// The heads' weight and bias gradients from gheads [2][B][z_pad], then their data gradient into gx = g(x pre-activation)
// = gmean Wm^T + glogvar Wl^T with wt = both kernels transposed, [2][z_pad][K].  dgrad_label may be null: no profile scope.
int32_t heads_backward(const Latent& h, const char* wgrad_label, const char* dgrad_label, const float* x, const float* gheads,
                       const float* wt, float* gx, float* partial, float* cs, float* grads, cudaStream_t s);
// z < z_pad: the zero-padded copies of the z-sized weights -- `heads`: both kernels [2][K][z_pad] at wp, both biases
// [2][z_pad] at bp; `dec`: the first decoder layer's kernel [z][N] at parameter offset dec_off, as [z_pad][N] at dp
void add_z_padding(RelayoutTable& t, const Latent& h, bool heads, int64_t wp, int64_t bp, bool dec, int64_t dec_off, int N,
                   int64_t dp);
// An rgb target that is the source itself (vae/train_vae.py:75) is read from the source's prepared, range-checked copy
bool target_is_source(const cpb_vae_config* c, const void* source, const void* target);
// [B, z_pad] latent rows of the workspace -> the caller's [B, z] rows of mean, logvar (heads) and z (zbuf), where given
int32_t copy_latents_out(const float* heads, const float* zbuf, int B, int z, int zp, float* mean, float* logvar, float* zout,
                         cudaStream_t s);

#pragma GCC visibility pop

}  // namespace cpb
