// HBM-bound kernels of the VAE step: frame preparation, transposed-conv output layer, sampling + KL,
// reconstruction loss (+ d loss / d logits), bias-gradient column sums, weight re-layout, TF-Adam.
#pragma once
#include "common.cuh"

namespace cpb {

// frames [npix, cin] (float32 in [0,1], or uint8 scaled by `scale`) -> [npix, 4] float32, zero padded.
// flags |= flag_bit when a value falls outside [0,1] (reference verify_range, vae/models.py:24-30).
int32_t launch_prep_frames(const void* src, int dtype, float scale, int cin, long long npix, float* dst,
                           int32_t* flags, int flag_bit, cudaStream_t stream);

// Output layer (tf conv2d_transpose 4x4 stride 2, 32 -> Ct channels): small [B,39,79,32] ->
// logits_p [B,80,160,4] (padded, bias added) and/or sigm [B,80,160,Ct] = sigmoid(logits).
int32_t launch_deconv4_fwd(const float* small, const float* w /*[4,4,Ct,32]*/, const float* bias, int batch,
                           int ct, float* logits_p, float* sigm, cudaStream_t stream);

// 3-channel edge layers (edge.cu): big4 = float4-per-pixel padded image [B,80,160,4], small [B,39,79,32], w = TF kernel [4,4,cb,32]
// gather: conv1 forward (mask == nullptr: bias + ReLU) / deconv4 data-gradient (mask != nullptr: ReLU mask, no bias)
// small_lo (nullable): also write small - trunc_tf32(small), the second TF32 operand of the tensor-core consumer
// cs_partial (optional, mask form only): [edge_gather_blocks(batch)][32] per-CTA column sums of `small` (bias gradient)
int32_t launch_edge_gather(const float* big4, int cb, const float* w, const float* bias, const float* mask,
                           float* small, float* small_lo, int batch, cudaStream_t stream, float* cs_partial = nullptr);
long long edge_gather_blocks(int batch);
// weight gradient: partial[edge_wgrad_ctas(batch)][16*cb][32]; reduce with launch_reduce_partials
int edge_wgrad_ctas(int batch);
int32_t launch_edge_wgrad(const float* big4, int cb, const float* small, int batch, float* partial, cudaStream_t stream);

// heads [2][B][z] (mean block, logvar block), eps [B,z] or nullptr -> zout [B,z], kl_rows [B],
// kl_active [B] (1 when the KL term of that row has a gradient, i.e. above the tolerance floor).
int32_t launch_reparam(const float* heads, const float* eps, int batch, int zdim, float kl_tolerance,
                       float* zout, float* kl_rows, float* kl_active, cudaStream_t stream);

// gz [B,z] -> gheads [2][B][z];  coef = beta * loss_scale / B
int32_t launch_reparam_bwd(const float* heads, const float* eps, const float* gz, const float* kl_active,
                           int batch, int zdim, float coef, float* gheads, cudaStream_t stream);

// logits_p, target_p [B,12800,4] -> frame_loss [B]; dlogits_p [B,12800,4] (nullable) = gscale * dl/dx
// frame_dsum (optional): [batch][4] per-frame channel sums of the gradient image (column-summed later = last layer's bias gradient)
int32_t launch_recon_loss(const float* logits_p, const float* target_p, int batch, int ct, int loss_type,
                          float gscale, float* frame_loss, float* dlogits_p, cudaStream_t stream, float* frame_dsum = nullptr);

// MlpVAE (flattened frames, no channel padding): dst[i] = src[i] * scale with the verify_range flag; y = sigmoid(x);
// reconstruction loss on unpadded [B, n] rows
int32_t launch_prep_flat(const void* src, int dtype, float scale, long long n, float* dst, int32_t* flags, int flag_bit, cudaStream_t stream);
int32_t launch_sigmoid(const float* x, float* y, long long n, cudaStream_t stream);
int32_t launch_recon_loss_flat(const float* logits, const float* target, int batch, int n, int loss_type, float gscale,
                               float* frame_loss, float* dlogits, cudaStream_t stream);

// losses[0] = scale * mean(frame_loss), losses[1] = scale * mean(kl_rows)
int32_t launch_finalize_losses(const float* frame_loss, const float* kl_rows, int batch, float scale,
                               float* losses, cudaStream_t stream);

// out[c] = sum_r g[r*pitch + c]  for c < c_real   (deterministic two-pass; scratch >= colsum_scratch_floats)
long long colsum_scratch_floats(long long rows, int pitch);
int32_t launch_colsum(const float* g, long long rows, int pitch, int c_real, float* out, float* scratch,
                      cudaStream_t stream);

// Weight re-layout jobs, all in one launch.
struct RelayoutJob {
    long long src_off, dst_off;   // float offsets into the params buffer / the relayout buffer
    int taps, rows, cols;         // source is [taps][rows][cols]
    int mode;                     // 0: transpose each tap -> [taps][cols][rows]
                                  // 1: pad rows -> [taps][rows_pad=4][cols]
    int rows_pad;
    long long count;              // destination elements
};
constexpr int kMaxRelayoutJobs = 12;   // (MlpVAE uses 6)
struct RelayoutTable {
    int njobs;
    long long total;
    RelayoutJob jobs[kMaxRelayoutJobs];
};
int32_t launch_relayout(const float* params, float* dst, const RelayoutTable& table, cudaStream_t stream);

// guard (nullable, device, one 32-bit word): when its bits are non-zero the update is skipped entirely (verify_range)
int32_t launch_adam(float* params, const float* grads, float* m, float* v, long long n, float* powers,
                    float lr, const float* lr_dev, float beta1, float beta2, float epsilon, cudaStream_t stream,
                    const void* guard = nullptr);

int32_t launch_fill_zero(float* p, long long n, cudaStream_t stream);

}  // namespace cpb
