// Weight-gradient GEMM (tf Conv2DBackpropFilter for conv AND transposed-conv layers, and the
// dense layers' x^T * g products):
//
//   gw[i, j] = sum_{m < M}  big[row(m) + tap_off[i / run] + i % run]  *  small[m * J + j]
//
// with m = (image, oy, ox) over the SMALL image grid, row(m) the stride-2 window origin in the BIG
// image, i = (kh, kw, cb) flattened exactly like the TF kernel [kh,kw,Cb,Cs] and j = cs.
// The reduction over M (up to 12.6 M positions) is split across CTAs; every split writes its own
// partial [I, J] block and reduce_partials() sums them in a fixed order (deterministic, no atomics).
#pragma once
#include "common.cuh"

namespace cpb {

struct WgradParams {
    const float* big;
    const float* small;
    float* partial;        // [splits][I][J]
    int batch;
    int Wb, big_pitch;     // big image width (pixels), floats per pixel
    long long big_img;     // floats per big image
    int Ho, Wo;            // small-image grid
    int sstride;           // 2 for conv layers, (ignored when Ho=Wo=1)
    int ntaps;             // kernel rows
    int run;               // floats per tap run (kW*Cb)
    long long tap_off[8];  // float offset of each tap run from the window origin
    int I, J;              // output rows / cols (J multiple of the tile's BJ)
    int splits;
    long long m_per_split; // multiple of 16
    int tc_variant;        // unused (kept for the cpb_debug_tc_wgrad signature)
    int passes;            // tensor-core path: 3 (3xTF32) or 1 (one TF32 pass, operands rounded to nearest)
};

// how many splits launch_wgrad will use for this problem (caller sizes `partial` with it)
int wgrad_pick_splits(int I, int J, long long M);
int32_t launch_wgrad(const WgradParams& p, cudaStream_t stream);
int32_t wgrad_init();

// tensor-core (wgmma, 3xTF32 or one TF32 pass) variant -- tc_wgrad.cu.  Same WgradParams; m_per_split must be a
// multiple of 32.
constexpr int kTcWaveCtas = 132;   // CTAs of the single split-K wave: one per SM of an H100 SXM
int32_t tc_wgrad_init();
bool tc_wgrad_supported(int I, int J, int run);
int tc_wgrad_pick_splits(int I, int J, long long M);
int32_t launch_tc_wgrad(const WgradParams& p, cudaStream_t stream);

// out[(t*c_real + c)*j_real + j] = sum_s partial[s][(t*c_pad + c)][j]   for c < c_real, j < j_real
int32_t launch_reduce_partials(const float* partial, int splits, int I, int J, int c_pad, int c_real, int j_real,
                               float* out, cudaStream_t stream);
// out[j][i] = sum_s partial[s][i][j]  (I, J multiples of 32): a weight gradient computed as its transpose
int32_t launch_reduce_partials_t(const float* partial, int splits, int I, int J, float* out, cudaStream_t stream);

}  // namespace cpb
