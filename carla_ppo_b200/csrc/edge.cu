// The two 3-channel "edge" layers of the ConvVAE (conv1: HxWx3 -> H1xW1x32 with H1 = H/2 - 1, W1 = W/2 - 1 -- 80x160x3 ->
// 39x79x32 by default -- and deconv4's gradient side).  The frame size is a run-time argument (FrameGeo).
// Their contraction is short (K = 4*4*Cb = 48, N = 32): the generic tap-GEMM spends its time in pipeline
// prologues, and per frame they only move ~360 KB -- they should run near the HBM roofline.  Dedicated kernels:
//
//   edge_gather_kernel : small[b,i,j,0:32] = epi( sum_{kh,kw,c<CB} big4[b,2i+kh,2j+kw,c] * W[kh,kw,c,0:32] )
//                        big4 is the float4-per-pixel padded image (prep_frames / recon_loss write it).
//                        conv1 forward (epi = bias+ReLU) and conv2d_transpose(deconv4) data-gradient (epi = ReLU mask).
//                        One thread = 4 horizontally adjacent output pixels x 16 channels: every weight float4 read
//                        from shared memory (warp-broadcast) feeds 16 FMAs, the padded channel is skipped.
//   edge_wgrad_kernel  : gw[kh,kw,c,j] = sum_{b,i,j'} big4[b,2i+kh,2j'+kw,c] * small[b,i,j',j]   (Conv2DBackpropFilter)
//                        One CTA walks output rows; per row it stages the 4 big rows and the small row in shared
//                        memory (cp.async), each warp accumulates the FULL [16*CB x 32] tile over its share of the
//                        row's positions with a 12x4 (or 4x4 when CB=1) register micro-tile, warps are combined
//                        through shared memory and each CTA writes one partial; reduce_partials sums them.
#include "elementwise.cuh"

namespace cpb {

namespace {

constexpr int SC = 32;   // small-side channels

// One thread = 4 horizontally adjacent output pixels x 16 of the 32 channels (lane parity picks the half).  The
// weights are read from shared memory as warp-broadcast LDS.128; such a load still writes 512 bytes of registers,
// i.e. occupies the 128 B/clk shared-memory return path for 4 cycles, so what matters is FMAs per LDS.128:
// 4 pixels x 4 channels = 16 (two pixels x 32 channels per thread gave 8 and left the kernel LDS-bound at twice
// its FMA time).
template <int CB, int EPI, int FH, int FW>   // EPI 0: bias + ReLU, 1: multiply by (mask > 0); FH, FW: FrameExtents
__global__ void __launch_bounds__(128)
edge_gather_kernel(const float4* __restrict__ big4, const float* __restrict__ w, const float* __restrict__ bias,
                   const float* __restrict__ mask, float* __restrict__ small, long long nwork, FrameGeo g,
                   float* __restrict__ cs_partial) {
    const FrameExtents<FH, FW> e(g);
    const int EH = e.H, EW = e.W, SH = e.H1, SW = e.W1;      // big image (pixels), small image
    __shared__ __align__(16) float ws[16 * CB * SC];
    for (int i = threadIdx.x; i < 16 * CB * SC; i += blockDim.x) ws[i] = w[i];
    __syncthreads();
    // cs_partial (mask form): this CTA's column sums of what it stores -> cs_partial[blockIdx.x][32] (the bias gradient of the layer
    // whose pre-activation gradient `small` is; summed over the CTAs by launch_colsum).  Fixed order: deterministic.
    __shared__ float csred[EPI == 1 ? 128 * 17 : 1];
    float csum[SC / 2];
#pragma unroll
    for (int j = 0; j < SC / 2; ++j) csum[j] = 0.f;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < nwork) {
    constexpr int NPX = 4;                               // output pixels per thread
    constexpr int HC = SC / 2;                           // channels per thread: the float4 groups 2*j4 + par, so that
    const int GW = (SW + NPX - 1) / NPX;                 // a lane pair's stores fill whole 32-byte sectors
    const int par = (int)(t & 1);
    const long long grp = t >> 1;
    const int gx = (int)(grp % GW);
    const int oy = (int)((grp / GW) % SH);
    const long long n = grp / (GW * SH);
    const int ox = gx * NPX;
    const int nvalid = SW - ox < NPX ? SW - ox : NPX;    // 4, or 3 in the last group of a row (W1 = 3 mod 4)

    float acc[NPX][HC];
#pragma unroll
    for (int q = 0; q < NPX; ++q)
#pragma unroll
        for (int j = 0; j < HC; ++j) acc[q][j] = 0.f;

    const float4* row0 = big4 + (n * EH + 2 * oy) * EW + 2 * ox;
    constexpr int NIN = 2 * (NPX - 1) + 4;               // 10 input pixels per kernel row
#pragma unroll
    for (int kh = 0; kh < 4; ++kh) {
        float4 in[NIN];
#pragma unroll
        for (int q = 0; q < NIN; ++q) in[q] = (2 * ox + q < EW) ? __ldg(row0 + kh * EW + q) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int kw = 0; kw < 4; ++kw) {
#pragma unroll
            for (int c = 0; c < CB; ++c) {
                float a[NPX];
#pragma unroll
                for (int q = 0; q < NPX; ++q) a[q] = c == 0 ? in[kw + 2 * q].x : (c == 1 ? in[kw + 2 * q].y : in[kw + 2 * q].z);
                const float* wr = &ws[((kh * 4 + kw) * CB + c) * SC + par * 4];
#pragma unroll
                for (int j4 = 0; j4 < HC / 4; ++j4) {
                    const float4 wv = *reinterpret_cast<const float4*>(wr + j4 * 8);
#pragma unroll
                    for (int q = 0; q < NPX; ++q) {
                        acc[q][j4 * 4 + 0] = fmaf(a[q], wv.x, acc[q][j4 * 4 + 0]);
                        acc[q][j4 * 4 + 1] = fmaf(a[q], wv.y, acc[q][j4 * 4 + 1]);
                        acc[q][j4 * 4 + 2] = fmaf(a[q], wv.z, acc[q][j4 * 4 + 2]);
                        acc[q][j4 * 4 + 3] = fmaf(a[q], wv.w, acc[q][j4 * 4 + 3]);
                    }
                }
            }
        }
    }
    const long long off = ((n * SH + oy) * SW + ox) * SC + par * 4;
#pragma unroll
    for (int q = 0; q < NPX; ++q) {
        if (q >= nvalid) break;
        const long long o = off + q * SC;
#pragma unroll
        for (int j4 = 0; j4 < HC / 4; ++j4) {
            float4 v = make_float4(acc[q][j4 * 4], acc[q][j4 * 4 + 1], acc[q][j4 * 4 + 2], acc[q][j4 * 4 + 3]);
            if (EPI == 0) {
                const float4 b = *reinterpret_cast<const float4*>(bias + par * 4 + j4 * 8);
                v.x = fmaxf(v.x + b.x, 0.f); v.y = fmaxf(v.y + b.y, 0.f); v.z = fmaxf(v.z + b.z, 0.f); v.w = fmaxf(v.w + b.w, 0.f);
            } else {
                const float4 mk = __ldg(reinterpret_cast<const float4*>(mask + o + j4 * 8));
                v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f; v.z = mk.z > 0.f ? v.z : 0.f; v.w = mk.w > 0.f ? v.w : 0.f;
            }
            *reinterpret_cast<float4*>(small + o + j4 * 8) = v;
            if (EPI == 1) { csum[j4 * 4] += v.x; csum[j4 * 4 + 1] += v.y; csum[j4 * 4 + 2] += v.z; csum[j4 * 4 + 3] += v.w; }
        }
    }
    }   // t < nwork
    if (EPI == 1 && cs_partial != nullptr) {
        // thread (parity par = tid & 1) holds the channels 8 * j4 + 4 * par + k at csum[4 * j4 + k]
#pragma unroll
        for (int j = 0; j < SC / 2; ++j) csred[threadIdx.x * 17 + j] = csum[j];
        __syncthreads();
        // two stages (16 + 4 terms per chain instead of one 64-term chain at the tail of every CTA), fixed order
        __shared__ float csq[4][SC];
        {
            const int c = threadIdx.x & (SC - 1), qd = threadIdx.x >> 5, par = (c >> 2) & 1, li = (c >> 3) * 4 + (c & 3);
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) a += csred[(qd * 32 + par + 2 * k) * 17 + li];
            csq[qd][c] = a;
        }
        __syncthreads();
        if (threadIdx.x < SC) cs_partial[(long long)blockIdx.x * SC + threadIdx.x] = (csq[0][threadIdx.x] + csq[1][threadIdx.x]) + (csq[2][threadIdx.x] + csq[3][threadIdx.x]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
constexpr int WG_WARPS = 8;
// shared-memory rows of edge_wgrad_kernel: a padded big row of W float4 pixels (the pitch + 4 puts the 4 kernel-row lane
// groups on different banks) and a small row of W1 x 32 floats (+ 32)
__host__ __device__ inline int wg_big_pitch(const FrameGeo& g) { return g.W * 4 + 4; }
__host__ __device__ inline int wg_small_pitch(const FrameGeo& g) { return g.W1 * SC + 32; }
// 2 x 4 big rows and 2 small rows (double buffer); at W = 48 the 8 big rows (1568 floats) still hold the combined
// [48 x 32] tile that reuses them
inline int wg_smem_bytes(const FrameGeo& g) { return (int)sizeof(float) * (8 * wg_big_pitch(g) + 2 * wg_small_pitch(g)); }

template <int CB, int FH, int FW>
__global__ void __launch_bounds__(WG_WARPS * 32)
edge_wgrad_kernel(const float* __restrict__ big4, const float* __restrict__ small, long long nrows, int rows_per_cta,
                  FrameGeo geo, float* __restrict__ partial) {
    // micro-tile: lane = (ig, jg): ig in [0, NI) owns TI rows of the [16*CB x 32] tile, jg in [0, 8) owns 4 columns
    constexpr int I = 16 * CB;                     // 48 or 16 rows: i = (kh*4 + kw)*CB + c
    constexpr int NI = 4, TI = I / NI;             // 12 or 4 rows per lane
    const FrameExtents<FH, FW> e(geo);
    const int EH = e.H, EW = e.W, SH = e.H1, SW = e.W1;
    const int BIG_ROW_FLOATS = EW * 4, SMALL_ROW_FLOATS = SW * SC;
    const int BIGP = EW * 4 + 4, SMALLP = SW * SC + 32;            // wg_big_pitch, wg_small_pitch
    // the 80x160 instantiation keeps its rows in static shared memory (41 KB), the run-time one in dynamic
    constexpr int kStaticFloats = FW ? 8 * (FW * 4 + 4) + 2 * ((FW / 2 - 1) * SC + 32) : 1;
    __shared__ __align__(16) float wg_static[kStaticFloats];
    extern __shared__ __align__(16) float wg_dynamic[];
    float* const wg_smem = FW ? wg_static : wg_dynamic;
    auto sbig = [&](int b) { return wg_smem + b * 4 * BIGP; };                 // [2][4 * BIGP]
    auto ssmall = [&](int b) { return wg_smem + 8 * BIGP + b * SMALLP; };      // [2][SMALLP]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ig = lane >> 3, jg = lane & 7;
    const long long r_begin = (long long)blockIdx.x * rows_per_cta;
    long long r_end = r_begin + rows_per_cta;
    if (r_end > nrows) r_end = nrows;

    float acc[TI][4];
#pragma unroll
    for (int a = 0; a < TI; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;

    auto stage_row = [&](int buf, long long r) {
        const long long n = r / SH;
        const int oy = (int)(r - n * SH);
        const float* gb = big4 + ((n * EH + 2 * oy) * EW) * 4;           // 4 consecutive padded rows of W float4 pixels
        for (int f = tid; f < 4 * BIG_ROW_FLOATS / 4; f += WG_WARPS * 32) {
            const int kh = f / (BIG_ROW_FLOATS / 4), q = f - kh * (BIG_ROW_FLOATS / 4);
            cp_async16(&sbig(buf)[kh * BIGP + q * 4], gb + f * 4, true);
        }
        const float* gs = small + r * SMALL_ROW_FLOATS;
        for (int f = tid; f < SMALL_ROW_FLOATS / 4; f += WG_WARPS * 32) cp_async16(&ssmall(buf)[f * 4], gs + f * 4, true);
    };

    if (r_begin < r_end) stage_row(0, r_begin);
    cp_async_commit();
    int buf = 0;
    for (long long r = r_begin; r < r_end; ++r, buf ^= 1) {
        if (r + 1 < r_end) stage_row(buf ^ 1, r + 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        // this warp's positions of the row: ox = warp, warp + 8, ...
        for (int ox = warp; ox < SW; ox += WG_WARPS) {
            const float4 g = *reinterpret_cast<const float4*>(&ssmall(buf)[ox * SC + jg * 4]);
            // lane group ig owns kernel row kh = ig: its TI = 4*CB values are the window row's 4 pixels x CB channels
            const float4* wp = reinterpret_cast<const float4*>(&sbig(buf)[ig * BIGP + 2 * ox * 4]);
            float a[TI];
#pragma unroll
            for (int kw = 0; kw < 4; ++kw) {
                const float4 px = wp[kw];
                a[kw * CB] = px.x;
                if (CB == 3) { a[kw * CB + 1] = px.y; a[kw * CB + 2] = px.z; }
            }
#pragma unroll
            for (int q = 0; q < TI; ++q) {
                acc[q][0] = fmaf(a[q], g.x, acc[q][0]); acc[q][1] = fmaf(a[q], g.y, acc[q][1]);
                acc[q][2] = fmaf(a[q], g.z, acc[q][2]); acc[q][3] = fmaf(a[q], g.w, acc[q][3]);
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();
    // ---- combine the 8 warps: each warp adds its tile into shared memory in turn (fixed order -> deterministic)
    float* tile = wg_smem;                                      // reuse: I*32 floats <= 1536 <= 8*BIGP
    __syncthreads();
    for (int w8 = 0; w8 < WG_WARPS; ++w8) {
        if (warp == w8) {
#pragma unroll
            for (int q = 0; q < TI; ++q)
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    float* dst = &tile[(ig * TI + q) * SC + jg * 4 + b];
                    *dst = (w8 == 0 ? 0.f : *dst) + acc[q][b];
                }
        }
        __syncthreads();
    }
    for (int f = tid; f < I * SC; f += WG_WARPS * 32) partial[(long long)blockIdx.x * I * SC + f] = tile[f];
}

}  // namespace

long long edge_gather_blocks(int batch, const FrameGeo& g) { return cdiv(2LL * batch * g.H1 * ((g.W1 + 3) / 4), 128); }

int32_t launch_edge_gather(const float* big4, int cb, const float* w, const float* bias, const float* mask,
                           float* small, int batch, const FrameGeo& g, cudaStream_t stream, float* cs_partial) {
    CPB_REQUIRE(cb == 1 || cb == 3, "edge_gather: channels must be 1 or 3");
    CPB_REQUIRE(cs_partial == nullptr || mask != nullptr, "edge_gather: column sums exist for the mask form only");
    const long long npairs = 2LL * batch * g.H1 * ((g.W1 + 3) / 4);  // (4-pixel group, channel half) work items
    if (npairs == 0) return CPB_OK;
    const unsigned blocks = (unsigned)cdiv(npairs, 128);
    const float4* b4 = reinterpret_cast<const float4*>(big4);
    auto launch = [&](auto kernel) {
        kernel<<<blocks, 128, 0, stream>>>(b4, w, mask ? nullptr : bias, mask, small, npairs, g, mask ? cs_partial : nullptr);
    };
    const bool fixed = is_default_frame(g);
    if (mask == nullptr) {
        if (cb == 3) launch(fixed ? edge_gather_kernel<3, 0, 80, 160> : edge_gather_kernel<3, 0, 0, 0>);
        else launch(fixed ? edge_gather_kernel<1, 0, 80, 160> : edge_gather_kernel<1, 0, 0, 0>);
    } else {
        if (cb == 3) launch(fixed ? edge_gather_kernel<3, 1, 80, 160> : edge_gather_kernel<3, 1, 0, 0>);
        else launch(fixed ? edge_gather_kernel<1, 1, 80, 160> : edge_gather_kernel<1, 1, 0, 0>);
    }
    CPB_LAUNCHED();
    return CPB_OK;
}

int edge_wgrad_ctas(int batch, const FrameGeo& g) {
    const long long nrows = (long long)batch * g.H1;
    long long ctas = 132 * 2;                     // two CTAs per SM of an H100 SXM
    if (ctas > nrows) ctas = nrows;
    return (int)(ctas < 1 ? 1 : ctas);
}

int32_t edge_init() {
    const FrameGeo widest = frame_geo(kMaxFrameSide, kMaxFrameSide);
    // (the 80x160 instantiations use 41 KB of static shared memory)
    CPB_CUDA(cudaFuncSetAttribute(edge_wgrad_kernel<3, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_bytes(widest)));
    CPB_CUDA(cudaFuncSetAttribute(edge_wgrad_kernel<1, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem_bytes(widest)));
    return CPB_OK;
}

int32_t launch_edge_wgrad(const float* big4, int cb, const float* small, int batch, const FrameGeo& g, float* partial,
                          cudaStream_t stream) {
    CPB_REQUIRE(cb == 1 || cb == 3, "edge_wgrad: channels must be 1 or 3");
    CPB_REQUIRE(g.W <= kMaxFrameSide, "edge_wgrad: frame width %d above %d", g.W, kMaxFrameSide);
    const long long nrows = (long long)batch * g.H1;
    if (nrows == 0) return CPB_OK;
    const int ctas = edge_wgrad_ctas(batch, g);
    const int rows_per_cta = (int)((nrows + ctas - 1) / ctas);
    const bool fixed = is_default_frame(g);
    const int smem = fixed ? 0 : wg_smem_bytes(g);
    auto launch = [&](auto kernel) { kernel<<<ctas, WG_WARPS * 32, smem, stream>>>(big4, small, nrows, rows_per_cta, g, partial); };
    if (cb == 3) launch(fixed ? edge_wgrad_kernel<3, 80, 160> : edge_wgrad_kernel<3, 0, 0>);
    else launch(fixed ? edge_wgrad_kernel<1, 80, 160> : edge_wgrad_kernel<1, 0, 0>);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
