// HBM-bound kernels of the VAE step: frame preparation, transposed-conv output layer, sampling + KL,
// reconstruction loss (+ d loss / d logits), bias-gradient column sums, weight re-layout, TF-Adam.
#pragma once
#include "common.cuh"

namespace cpb {

// The frame-resolution geometry of the ConvVAE: the frame [H, W] and conv1's output [H1, W1] = [H/2 - 1, W/2 - 1]
// (4x4 stride-2 VALID).  Legal frames have H and W multiples of 16 in [48, kMaxFrameSide]: then W1 = 3 (mod 4) and W/2
// is a multiple of 8, the row structure the edge and deconv4 kernels rely on.
struct FrameGeo { int H, W, H1, W1; };
constexpr int kMaxFrameSide = 512;
inline FrameGeo frame_geo(int H, int W) { return FrameGeo{H, W, H / 2 - 1, W / 2 - 1}; }
// The frame-resolution kernels take the frame size at run time (template arguments FH = FW = 0), or fixed at compile time
// for the reference's 80x160 (FH, FW = 80, 160), which the launchers pick for that geometry: with the extents known the
// index arithmetic folds, and the 80x160 step measured 1.3 % (3xTF32) / 2.1 % (TF32) faster on an H100 than with the
// run-time kernels (README, "Frame size").  Both compute the same values in the same order.
template <int FH, int FW>
struct FrameExtents {
    int H, W, H1, W1;
    __host__ __device__ explicit FrameExtents(const FrameGeo& g)
        : H(FH ? FH : g.H), W(FW ? FW : g.W), H1(FH ? FH / 2 - 1 : g.H1), W1(FW ? FW / 2 - 1 : g.W1) {}
};
inline bool is_default_frame(const FrameGeo& g) { return g.H == 80 && g.W == 160; }

// frames [npix, cin] (float32 in [0,1], or uint8 scaled by `scale`) -> [npix, 4] float32, zero padded.
// flags |= flag_bit when a value falls outside [0,1] (reference verify_range, vae/models.py:24-30).
int32_t launch_prep_frames(const void* src, int dtype, float scale, int cin, long long npix, float* dst,
                           int32_t* flags, int flag_bit, cudaStream_t stream);

// Output layer (tf conv2d_transpose 4x4 stride 2, 32 -> Ct channels): small [B,H1,W1,32] ->
// logits_p [B,H,W,4] (padded, bias added) and/or sigm [B,H,W,Ct] = sigmoid(logits).
int32_t launch_deconv4_fwd(const float* small, const float* w /*[4,4,Ct,32]*/, const float* bias, int batch,
                           int ct, const FrameGeo& g, float* logits_p, float* sigm, cudaStream_t stream);

// 3-channel edge layers (edge.cu): big4 = float4-per-pixel padded image [B,H,W,4], small [B,H1,W1,32], w = TF kernel [4,4,cb,32]
// gather: conv1 forward (mask == nullptr: bias + ReLU) / deconv4 data-gradient (mask != nullptr: ReLU mask, no bias)
// cs_partial (optional, mask form only): [edge_gather_blocks(batch, g)][32] per-CTA column sums of `small` (bias gradient)
int32_t launch_edge_gather(const float* big4, int cb, const float* w, const float* bias, const float* mask,
                           float* small, int batch, const FrameGeo& g, cudaStream_t stream, float* cs_partial = nullptr);
long long edge_gather_blocks(int batch, const FrameGeo& g);
// weight gradient: partial[edge_wgrad_ctas(batch, g)][16*cb][32]; reduce with launch_reduce_partials.  edge_init opts the
// kernel in to the shared memory of the widest legal frame (once per device).
int32_t edge_init();
int edge_wgrad_ctas(int batch, const FrameGeo& g);
int32_t launch_edge_wgrad(const float* big4, int cb, const float* small, int batch, const FrameGeo& g, float* partial,
                          cudaStream_t stream);

// heads [2][B][pitch] (mean block, logvar block), eps [B,zdim] or nullptr -> zout [B,pitch], kl_rows [B],
// kl_active [B] (1 when the KL term of that row has a gradient, i.e. above the tolerance floor).  The KL sums the
// zdim real columns; zout's columns zdim..pitch-1 are written as 0.
int32_t launch_reparam(const float* heads, const float* eps, int batch, int zdim, int pitch, float kl_tolerance,
                       float* zout, float* kl_rows, float* kl_active, cudaStream_t stream);

// gz [B,pitch] -> gheads [2][B][pitch] (columns zdim..pitch-1 written as 0);  coef = beta * loss_scale / B
int32_t launch_reparam_bwd(const float* heads, const float* eps, const float* gz, const float* kl_active,
                           int batch, int zdim, int pitch, float coef, float* gheads, cudaStream_t stream);

// [rows, src_pitch] -> [rows, dst_pitch]: copies min(src_pitch, dst_pitch) columns, zero-fills the rest of each row
// (the latent boundary: callers' [B, z] rows <-> the library's [B, z_pad] rows).  Pitches are multiples of 4.
int32_t launch_pitch_copy(const float* src, int src_pitch, float* dst, int dst_pitch, int rows, cudaStream_t stream);

// logits_p, target_p [B,npix,4] -> frame_loss [B]; dlogits_p [B,npix,4] (nullable) = gscale * dl/dx
// frame_dsum (optional): [batch][4] per-frame channel sums of the gradient image (column-summed later = last layer's bias gradient)
int32_t launch_recon_loss(const float* logits_p, const float* target_p, int batch, int npix, int ct, int loss_type,
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
    int mode;                     // 0: transpose each tap -> [taps][cols_pad][rows_pad]
                                  // 1: copy each tap -> [taps][rows_pad][cols_pad]
    int rows_pad, cols_pad;       // >= rows, cols; the padding is zero-filled
    long long count;              // destination elements
};
constexpr int kMaxRelayoutJobs = 16;   // (the ConvVAE step uses up to 12)
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
