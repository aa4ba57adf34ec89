// Tap-GEMM: the one fp32 kernel family behind every dense contraction of the ConvVAE
// (conv forward, transposed-conv forward, both data-gradients and the dense layers).
//
//   dst[pix(m), n] = epilogue( sum_{tap} sum_{c < C}  src[row(m) + tap.src_off + c] * W[tap.w_off + c*ldw + n] )
//
// A "tap" is one contiguous run of C source floats per output position plus the [C x N] weight
// block that multiplies it:
//   * gather form (tf Conv2D fwd, conv2d_transpose data-gradient): one tap per kernel row kh, the run
//     is the (kw, cb) span of the stride-2 window -- always in bounds (VALID padding);
//   * scatter form (conv2d_transpose fwd = Conv2DBackpropInput, Conv2D data-gradient): outputs are
//     split into the 4 (y%2, x%2) parity classes; inside a class the layer is a stride-1 correlation
//     with the taps {kh = py+2j, kw = px+2i}, bounds-checked (zero-filled) at the image border;
//   * dense layers are 1x1 images with one tap (two for the fused heads' input gradient).
#pragma once
#include "common.cuh"

namespace cpb {

constexpr int kMaxTaps = 25;

struct Tap {
    int dy, dx;           // source pixel displacement (bounds check only)
    long long src_off;    // float offset added to the row base
    long long w_off;      // float offset of this tap's [C x N] weight block
};

struct TapClass {
    int ntaps;
    int py, px;           // destination parity offset (0 for gather form)
    int Ho, Wo;           // output grid of this class
    Tap taps[kMaxTaps];
};

struct TapGemmParams {
    const float* src;
    const float* wmat;
    const float* bias;    // [N] or nullptr
    const float* mask;    // same shape as dst: out *= (mask > 0), or nullptr
    float* dst;
    int batch;
    int Hs, Ws;           // source image extent (pixels)
    int src_pitch;        // floats per source pixel
    long long src_img;    // floats per source image
    int sstride;          // source pixels per output step (2 gather, 1 scatter/dense)
    int C;                // floats per tap run (multiple of 16)
    int N;                // output channels handled per y-batch (multiple of the tile's BN)
    int ldw;              // weight row stride in floats
    int Hd, Wd;           // destination image extent
    int dstride;          // destination pixels per output step (1 gather, 2 scatter)
    int dst_pitch;        // floats per destination pixel
    long long dst_img;    // floats per destination image
    int relu;
    int check;            // bounds-check taps (scatter form)
    int nclass;           // 1 or 4
    int ybatch;           // independent problems sharing src (fused heads): 1 or 2
    long long w_ystride, bias_ystride, dst_ystride;
    int ksplit;           // >= 1; > 1 (SIMT path, dense layers only): the reduction is split over gridDim.z into
    float* kpartial;      // kpartial[ksplit][kpartial_stride] raw partial results, then reduced with the epilogue
    long long kpartial_stride;
    // tensor-core path only: K-major per-tap [N][C] weight blocks, pre-split into hi / lo (tc_tapgemm.cu)
    const float* wk_hi;
    const float* wk_lo;
    const float* src_lo;  // tensor-core path only: lo plane of src (x - trunc_tf32(x)), same indexing as src
    float* dst_lo;        // tensor-core path only: if set, the epilogue also writes the lo plane of dst (for the next layer)
    // tensor-core path only: quad-fused scatter form.  One GEMM row = one 2x2 output quad (qy, qx); the N axis is
    // (parity class, cb) = 4*quad_cb columns; cls[0] holds the union window taps (2x2 for k=4, 3x3 for k=5) and the
    // weight blocks carry zeros where a class does not use a tap.  The A tile is loaded once for all four classes.
    int quad;
    int quad_cb;
    int quad_lcb;         // log2(quad_cb), set by the launcher
    int cluster;          // tensor-core path: CTAs per cluster (set by the launcher)
    int debug;            // tensor-core path: timing decomposition (CPB_TC_DEBUG): 2 no A copies, 4 A copies zero-fill only, 8 no weight copies
    TapClass cls[4];
};

// Enqueue; picks the tile shape from N and the row count.
int32_t launch_tapgemm(const TapGemmParams& p, cudaStream_t stream);
constexpr int kMaxKSplit = 8;
// k-split factor for a dense [rows x K] x [K x N] layer with N % 64 == 0 (1 = do not split)
int tapgemm_pick_ksplit(int rows, int N, int ybatch, int K);
// One-time opt-in for >48 KB dynamic shared memory (called from the API layer).
int32_t tapgemm_init();

// ---- tensor-core (wgmma, 3xTF32) variant of the same contraction -------------------------------------------------
struct TcWeightJob {
    long long src_off;          // float offset of the TF kernel [k,k,Cb,Cs] in the parameter buffer
    long long dst_hi, dst_lo;   // float offset of the operand (2 * taps * N * C floats, hi and lo interleaved by block) / unused
    int mode;                   // logical operand per tap [N][C]:  0: plain K-major matrix; 1: gather form [kh][cs][kw*Cb+cb];
                                // 2: quad scatter form [j][i][class*Cb+cb][cs], window w = (k+1)/2, zero where unused
    int k, cb, cs;
    int N, C;                   // logical rows / reduction length per tap
    long long count;
};
// rows of the N axis handled per CTA tile (also fixes the block size of the stored operand); at most 64, because each
// consumer thread holds 1.5 x BN fp32 accumulators in registers
__host__ __device__ constexpr int tc_bn(int N) { return N % 64 == 0 ? 64 : 32; }
constexpr int kMaxTcWeightJobs = 12;
struct TcWeightTable {
    int njobs;
    long long total;
    TcWeightJob jobs[kMaxTcWeightJobs];
};
int32_t tc_tapgemm_init();
bool tc_tapgemm_supported(const TapGemmParams& p);
int32_t launch_tc_tapgemm(const TapGemmParams& p, cudaStream_t stream);
// lo[i] = x[i] - (x[i] with the 13 low mantissa bits cleared), count floats (multiple of 4)
int32_t launch_lo_plane(const float* x, float* lo, long long count, cudaStream_t stream);
int32_t launch_tc_weights(const float* params, float* dst, const TcWeightTable& table, cudaStream_t stream);

}  // namespace cpb
