// HBM-bound / small kernels of the VAE step (see elementwise.cuh).
#include "elementwise.cuh"

namespace cpb {

namespace {

// ------------------------------------------------------------------------------------------
// frame preparation: [npix, CIN] (f32 or u8) -> [npix, 4] f32, range check
// ------------------------------------------------------------------------------------------
template <typename T, int CIN>
__global__ void prep_frames_kernel(const T* __restrict__ src, float scale, long long npix,
                                   float* __restrict__ dst, int32_t* flags, int flag_bit) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (p < npix) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int c = 0; c < CIN; ++c) {
            const float x = (float)src[p * CIN + c] * scale;
            v[c] = x;
            bad = bad || !(x >= 0.f && x <= 1.f);
        }
        reinterpret_cast<float4*>(dst)[p] = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (flags != nullptr && __any_sync(0xffffffffu, bad)) {
        if ((threadIdx.x & 31) == 0) atomicOr(flags, flag_bit);
    }
}

// flat variant (MlpVAE: tf.layers.flatten of the NHWC frame, no channel padding): dst[i] = src[i] * scale, range check
template <typename T>
__global__ void prep_flat_kernel(const T* __restrict__ src, float scale, long long n, float* __restrict__ dst, int32_t* flags, int flag_bit) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (i < n) {
        const float x = (float)src[i] * scale;
        dst[i] = x;
        bad = !(x >= 0.f && x <= 1.f);
    }
    if (flags != nullptr && __any_sync(0xffffffffu, bad)) {
        if ((threadIdx.x & 31) == 0) atomicOr(flags, flag_bit);
    }
}

__global__ void sigmoid_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = 1.f / (1.f + expf(-x[i]));
}

// ------------------------------------------------------------------------------------------
// output layer: conv2d_transpose 4x4 s2, 32 -> CT channels.
// ------------------------------------------------------------------------------------------
// One thread = NQ horizontally adjacent 2x2 output quads.  Every weight float4 read from shared memory
// (warp-broadcast LDS.128, which occupies the 128 B/clk return path for 4 cycles) feeds NQ x 4 FMAs.
template <int CT, int NQ, int FH, int FW>   // FH, FW: FrameExtents
__global__ void __launch_bounds__(128)
deconv4_fwd_kernel(const float* __restrict__ small, const float* __restrict__ w, const float* __restrict__ bias,
                   long long nwork, FrameGeo g, float* __restrict__ logits_p, float* __restrict__ sigm) {
    // small [HS, WS] = [H1, W1]; output quads [QH, QW] = [H/2, W/2] (W/2 is a multiple of 8: NQ divides a quad row)
    constexpr int CS = 32;
    const FrameExtents<FH, FW> e(g);
    const int HS = e.H1, WS = e.W1, QH = e.H / 2, QW = e.W / 2, HB = e.H, WB = e.W, PW = QW / NQ;
    __shared__ __align__(16) float ws[16 * CT * CS];
    for (int i = threadIdx.x; i < 16 * CT * CS; i += blockDim.x) ws[i] = w[i];
    __syncthreads();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nwork) return;
    const int qx0 = (int)(t % PW) * NQ;
    const int qy = (int)((t / PW) % QH);
    const long long n = t / (PW * QH);

    float acc[NQ][2][2][CT];     // [quad][py][px][c]
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int c = 0; c < CT; ++c) acc[q][a][b][c] = bias[c];

#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int iy = qy - j;
        if (iy < 0 || iy >= HS) continue;
        const float* rowp = small + ((n * HS + iy) * WS) * CS;
        // input pixels p = qx0-1 .. qx0+NQ-1 ; quad q uses pixel (q + 1 - i) for tap column i
        bool pv[NQ + 1];
#pragma unroll
        for (int p = 0; p < NQ + 1; ++p) pv[p] = (unsigned)(qx0 - 1 + p) < (unsigned)WS;
#pragma unroll
        for (int c4 = 0; c4 < CS / 4; ++c4) {
            float4 x[NQ + 1];
#pragma unroll
            for (int p = 0; p < NQ + 1; ++p)
                x[p] = pv[p] ? __ldg(reinterpret_cast<const float4*>(rowp + (qx0 - 1 + p) * CS) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int py = 0; py < 2; ++py)
#pragma unroll
                    for (int px = 0; px < 2; ++px) {
                        const int tap = (py + 2 * j) * 4 + (px + 2 * i);
#pragma unroll
                        for (int c = 0; c < CT; ++c) {
                            const float4 wv = *reinterpret_cast<const float4*>(&ws[(tap * CT + c) * CS + c4 * 4]);
#pragma unroll
                            for (int q = 0; q < NQ; ++q) {
                                const float4 xv = x[q + 1 - i];
                                float s = acc[q][py][px][c];
                                s = fmaf(xv.x, wv.x, s); s = fmaf(xv.y, wv.y, s);
                                s = fmaf(xv.z, wv.z, s); s = fmaf(xv.w, wv.w, s);
                                acc[q][py][px][c] = s;
                            }
                        }
                    }
        }
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int py = 0; py < 2; ++py)
#pragma unroll
            for (int px = 0; px < 2; ++px) {
                const long long pix = (n * HB + 2 * qy + py) * WB + 2 * (qx0 + q) + px;
                if (logits_p != nullptr) {
                    float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int c = 0; c < CT; ++c) v[c] = acc[q][py][px][c];
                    reinterpret_cast<float4*>(logits_p)[pix] = make_float4(v[0], v[1], v[2], v[3]);
                }
                if (sigm != nullptr) {
#pragma unroll
                    for (int c = 0; c < CT; ++c) sigm[pix * CT + c] = 1.f / (1.f + expf(-acc[q][py][px][c]));
                }
            }
}

// ------------------------------------------------------------------------------------------
// sampling + KL: one warp per row
// ------------------------------------------------------------------------------------------
__global__ void reparam_kernel(const float* __restrict__ heads, const float* __restrict__ eps, int batch,
                               int zdim, int pitch, float kl_floor, int use_floor, float* __restrict__ zout,
                               float* __restrict__ kl_rows, float* __restrict__ kl_active) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= batch) return;
    const float* mu = heads + (long long)row * pitch;
    const float* lv = heads + (long long)batch * pitch + (long long)row * pitch;
    float s = 0.f;
    for (int j = lane; j < zdim; j += 32) {
        const float m = mu[j], l = lv[j];
        const float z = eps != nullptr ? fmaf(eps[(long long)row * zdim + j], expf(0.5f * l), m) : m;
        zout[(long long)row * pitch + j] = z;
        s += 1.f + l - m * m - expf(l);
    }
    for (int j = zdim + lane; j < pitch; j += 32) zout[(long long)row * pitch + j] = 0.f;
    s = warp_sum(s);
    if (lane == 0) {
        float kl = -0.5f * s;
        float active = 1.f;
        if (use_floor) {
            active = kl >= kl_floor ? 1.f : 0.f;   // tf.maximum routes the gradient to kl when kl >= floor
            kl = fmaxf(kl, kl_floor);
        }
        kl_rows[row] = kl;
        kl_active[row] = active;
    }
}

__global__ void reparam_bwd_kernel(const float* __restrict__ heads, const float* __restrict__ eps,
                                   const float* __restrict__ gz, const float* __restrict__ kl_active,
                                   int batch, int zdim, int pitch, float coef, float* __restrict__ gheads) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)batch * pitch;
    if (idx >= n) return;
    const int row = (int)(idx / pitch);
    const int col = (int)(idx - (long long)row * pitch);
    if (col >= zdim) {
        gheads[idx] = 0.f;
        gheads[n + idx] = 0.f;
        return;
    }
    const float m = heads[idx], l = heads[n + idx];
    const float g = gz[idx];
    const float a = kl_active[row] * coef;
    const float e = eps != nullptr ? eps[(long long)row * zdim + col] : 0.f;
    gheads[idx] = fmaf(a, m, g);
    gheads[n + idx] = g * (0.5f * e * expf(0.5f * l)) + a * 0.5f * (expf(l) - 1.f);
}

// dst[r, c] = c < src_pitch ? src[r, c] : 0   for c < dst_pitch (both pitches multiples of 4)
__global__ void pitch_copy_kernel(const float4* __restrict__ src, int src_p4, float4* __restrict__ dst, int dst_p4,
                                  long long n4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const long long r = i / dst_p4;
    const int c = (int)(i - r * dst_p4);
    dst[i] = c < src_p4 ? src[r * src_p4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// ------------------------------------------------------------------------------------------
// reconstruction loss: one CTA per frame
// ------------------------------------------------------------------------------------------
template <int LOSS>
__device__ __forceinline__ void loss_elem(float x, float y, float& val, float& dx) {
    const float s = 1.f / (1.f + expf(-x));
    if (LOSS == CPB_LOSS_MSE) {
        const float d = y - s;
        val = d * d;
        dx = -2.f * d * s * (1.f - s);
    } else if (LOSS == CPB_LOSS_BCE) {
        val = fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
        dx = s - y;
    } else {
        const float e = 1e-10f;
        val = -(y * logf(e + s) + (1.f - y) * logf(e + 1.f - s));
        dx = -(y / (e + s) - (1.f - y) / (e + 1.f - s)) * s * (1.f - s);
    }
}

template <int LOSS, int CT>
__global__ void __launch_bounds__(256)
recon_loss_kernel(const float4* logits_p, const float4* __restrict__ target_p, int npix, float gscale,
                  float* __restrict__ frame_loss, float4* dlogits_p, float* __restrict__ frame_dsum) {
    // logits_p and dlogits_p MAY ALIAS (the training path overwrites the logits with d loss / d logits in place): neither
    // is __restrict__, each element is read before it is written by the same thread.
    // frame_dsum (optional): [batch][4] per-frame channel sums of d loss / d logits -- the last layer's bias gradient is their
    // column sum, which saves a separate pass over the [B, H, W, 4] gradient image
    const long long base = (long long)blockIdx.x * npix;
    float sum = 0.f;
    float ds[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = threadIdx.x; p < npix; p += blockDim.x) {
        const float4 l = logits_p[base + p];
        const float4 y = target_p[base + p];
        const float lv[4] = {l.x, l.y, l.z, l.w};
        const float yv[4] = {y.x, y.y, y.z, y.w};
        float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            float val, dx;
            loss_elem<LOSS>(lv[c], yv[c], val, dx);
            sum += val;
            d[c] = dx * gscale;
            ds[c] += d[c];
        }
        if (dlogits_p != nullptr) dlogits_p[base + p] = make_float4(d[0], d[1], d[2], d[3]);
    }
    __shared__ float red[5][8];
    sum = warp_sum(sum);
    if (frame_dsum != nullptr) {
#pragma unroll
        for (int c = 0; c < 4; ++c) ds[c] = warp_sum(ds[c]);
    }
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = sum;
#pragma unroll
        for (int c = 0; c < 4; ++c) red[1 + c][threadIdx.x >> 5] = ds[c];
    }
    __syncthreads();
    if (threadIdx.x < 5 && (threadIdx.x == 0 || frame_dsum != nullptr)) {
        float t = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[threadIdx.x][i];
        if (threadIdx.x == 0) frame_loss[blockIdx.x] = t;
        else frame_dsum[(long long)blockIdx.x * 4 + threadIdx.x - 1] = t;
    }
}

__global__ void finalize_losses_kernel(const float* __restrict__ frame_loss, const float* __restrict__ kl_rows,
                                       int batch, float scale, float* __restrict__ losses) {
    __shared__ double red[2][32];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < batch; i += blockDim.x) {
        a += (double)frame_loss[i];
        b += (double)kl_rows[i];
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0.0, tb = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { ta += red[0][i]; tb += red[1][i]; }
        losses[0] = (float)(ta / batch * scale);
        losses[1] = (float)(tb / batch * scale);
    }
}

// ------------------------------------------------------------------------------------------
// column sums (bias gradients): pass 1 -> partial[blocks][pitch]
// ------------------------------------------------------------------------------------------
constexpr int kColsumMaxBlocks = 132 * 8;   // 8 blocks per SM of an H100 SXM
// number of row-chunk blocks; block b sums the row tiles b, b + nblocks, b + 2 nblocks, ... (a tile = the rows one
// pass of the block covers), so that at any moment the resident blocks read one contiguous stretch of memory.
// (Giving each block ONE contiguous range made the ~1200 concurrent streams start 1.3 MB apart and ran the
// [12.6M x 32] sums at a quarter of the HBM rate.)
static long long colsum_blocks(long long rows, int pitch) {
    const int c4_total = pitch >> 2;
    const int cw = c4_total < 256 ? c4_total : 256;
    const long long tiles = (rows + (256 / cw) - 1) / (256 / cw);
    long long nb = (tiles + 7) / 8;                        // at least 8 tiles per block
    if (nb > kColsumMaxBlocks) nb = kColsumMaxBlocks;
    return nb < 1 ? 1 : nb;
}

__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ g, long long rows, int pitch, float* __restrict__ partial) {
    // blockIdx.x: row-tile residue; blockIdx.y: chunk of 256 float4 columns
    const int c4_total = pitch >> 2;
    const int cw = c4_total < 256 ? c4_total : 256;        // float4 columns handled by this block
    const int lanes_r = 256 / cw;                           // rows per tile
    const int cc = threadIdx.x % cw;
    const int rr = threadIdx.x / cw;
    const int col4 = blockIdx.y * 256 + cc;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (col4 < c4_total && rr < lanes_r) {
        // 8 independent loads in flight per thread; the summation order is fixed (deterministic)
        const float4* base = reinterpret_cast<const float4*>(g) + col4;
        const long long p4 = pitch >> 2;
        const long long step = (long long)gridDim.x * lanes_r;
        long long r = (long long)blockIdx.x * lanes_r + rr;
        float4 a2 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (; r + 7 * step < rows; r += 8 * step) {
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = __ldg(base + (r + u * step) * p4);
#pragma unroll
            for (int u = 0; u < 8; u += 2) {
                acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
                a2.x += v[u + 1].x; a2.y += v[u + 1].y; a2.z += v[u + 1].z; a2.w += v[u + 1].w;
            }
        }
        for (; r < rows; r += step) {
            const float4 v = __ldg(base + r * p4);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        acc.x += a2.x; acc.y += a2.y; acc.z += a2.z; acc.w += a2.w;
    }
    __shared__ float4 red[256];
    red[threadIdx.x] = acc;
    __syncthreads();
    if (rr == 0 && col4 < c4_total) {
        for (int k = 1; k < lanes_r; ++k) {
            const float4 v = red[k * cw + cc];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        reinterpret_cast<float4*>(partial + (long long)blockIdx.x * pitch)[col4] = acc;
    }
}

// one warp per column: lanes stride over the row-chunk partials, fixed-order shuffle reduction
__global__ void colsum_final_kernel(const float* __restrict__ partial, int nblocks, int pitch, int c_real,
                                    float* __restrict__ out) {
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (c >= c_real) return;
    float s = 0.f;
    for (int b = lane; b < nblocks; b += 32) s += partial[(long long)b * pitch + c];
    s = warp_sum(s);
    if (lane == 0) out[c] = s;
}

// ------------------------------------------------------------------------------------------
// weight re-layout
// ------------------------------------------------------------------------------------------
__global__ void relayout_kernel(const float* __restrict__ params, float* __restrict__ dst,
                                const __grid_constant__ RelayoutTable t) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= t.total) return;
    int j = 0;
    while (j < t.njobs - 1 && idx >= t.jobs[j].count) { idx -= t.jobs[j].count; ++j; }
    const RelayoutJob& job = t.jobs[j];
    int r, c, tap;
    if (job.mode == 0) {
        // dst [taps][cols_pad][rows_pad]
        r = (int)(idx % job.rows_pad);
        const long long rest = idx / job.rows_pad;
        c = (int)(rest % job.cols_pad);
        tap = (int)(rest / job.cols_pad);
    } else {
        // dst [taps][rows_pad][cols_pad]
        c = (int)(idx % job.cols_pad);
        const long long rest = idx / job.cols_pad;
        r = (int)(rest % job.rows_pad);
        tap = (int)(rest / job.rows_pad);
    }
    dst[job.dst_off + idx] = r < job.rows && c < job.cols ? params[job.src_off + ((long long)tap * job.rows + r) * job.cols + c] : 0.f;
}

// ------------------------------------------------------------------------------------------
// TF ApplyAdam
// ------------------------------------------------------------------------------------------
__global__ void adam_kernel(float4* __restrict__ p, const float4* __restrict__ g, float4* __restrict__ m,
                            float4* __restrict__ v, long long n4, const float* __restrict__ powers, float lr,
                            const float* __restrict__ lr_dev, float beta1, float beta2, float epsilon,
                            const uint32_t* __restrict__ guard) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    if (guard != nullptr && guard[0] != 0u) return;     // verify_range tripped: the reference's tf.Assert aborts BEFORE the update
    const float lr_t = lr_dev != nullptr ? lr_dev[0] : lr;
    const float alpha = lr_t * sqrtf(1.f - powers[1]) / (1.f - powers[0]);
    const float omb1 = 1.f - beta1, omb2 = 1.f - beta2;
    const float4 gv = g[i];
    float4 mv = m[i], vv = v[i], pv = p[i];
    mv.x += (gv.x - mv.x) * omb1; mv.y += (gv.y - mv.y) * omb1; mv.z += (gv.z - mv.z) * omb1; mv.w += (gv.w - mv.w) * omb1;
    vv.x += (gv.x * gv.x - vv.x) * omb2; vv.y += (gv.y * gv.y - vv.y) * omb2;
    vv.z += (gv.z * gv.z - vv.z) * omb2; vv.w += (gv.w * gv.w - vv.w) * omb2;
    pv.x -= (mv.x * alpha) / (sqrtf(vv.x) + epsilon); pv.y -= (mv.y * alpha) / (sqrtf(vv.y) + epsilon);
    pv.z -= (mv.z * alpha) / (sqrtf(vv.z) + epsilon); pv.w -= (mv.w * alpha) / (sqrtf(vv.w) + epsilon);
    m[i] = mv; v[i] = vv; p[i] = pv;
}

__global__ void adam_powers_kernel(float* powers, float beta1, float beta2, const uint32_t* __restrict__ guard) {
    if (guard != nullptr && guard[0] != 0u) return;
    powers[0] *= beta1;
    powers[1] *= beta2;
}

__global__ void fill_zero_kernel(float4* p, long long n4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n4) p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

}  // namespace

// ============================================================================================
int32_t launch_prep_frames(const void* src, int dtype, float scale, int cin, long long npix, float* dst,
                           int32_t* flags, int flag_bit, cudaStream_t stream) {
    CPB_REQUIRE(cin == 1 || cin == 3, "prep_frames: cin must be 1 or 3");
    const unsigned blocks = (unsigned)cdiv(npix, 256);
    if (blocks == 0) return CPB_OK;
    if (dtype == CPB_FRAME_F32) {
        if (cin == 3) prep_frames_kernel<float, 3><<<blocks, 256, 0, stream>>>((const float*)src, scale, npix, dst, flags, flag_bit);
        else prep_frames_kernel<float, 1><<<blocks, 256, 0, stream>>>((const float*)src, scale, npix, dst, flags, flag_bit);
    } else if (dtype == CPB_FRAME_U8) {
        if (cin == 3) prep_frames_kernel<uint8_t, 3><<<blocks, 256, 0, stream>>>((const uint8_t*)src, scale, npix, dst, flags, flag_bit);
        else prep_frames_kernel<uint8_t, 1><<<blocks, 256, 0, stream>>>((const uint8_t*)src, scale, npix, dst, flags, flag_bit);
    } else {
        CPB_REQUIRE(false, "prep_frames: unknown frame dtype %d", dtype);
    }
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_deconv4_fwd(const float* small, const float* w, const float* bias, int batch, int ct, const FrameGeo& g,
                           float* logits_p, float* sigm, cudaStream_t stream) {
    constexpr int nq = 4;                                          // 8 quads per thread measured 2x slower (254 registers)
    CPB_REQUIRE(g.W % (2 * nq) == 0, "deconv4: frame width %d is not a multiple of %d", g.W, 2 * nq);
    const long long npairs = (long long)batch * (g.H / 2) * (g.W / 2 / nq);   // groups of nq horizontally adjacent 2x2 output quads
    if (npairs == 0) return CPB_OK;
    const unsigned blocks = (unsigned)cdiv(npairs, 128);
    CPB_REQUIRE(ct == 1 || ct == 3, "deconv4: target_channels must be 1 or 3");
    auto launch = [&](auto kernel) { kernel<<<blocks, 128, 0, stream>>>(small, w, bias, npairs, g, logits_p, sigm); };
    const bool fixed = is_default_frame(g);
    if (ct == 3) launch(fixed ? deconv4_fwd_kernel<3, nq, 80, 160> : deconv4_fwd_kernel<3, nq, 0, 0>);
    else launch(fixed ? deconv4_fwd_kernel<1, nq, 80, 160> : deconv4_fwd_kernel<1, nq, 0, 0>);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_reparam(const float* heads, const float* eps, int batch, int zdim, int pitch, float kl_tolerance,
                       float* zout, float* kl_rows, float* kl_active, cudaStream_t stream) {
    if (batch == 0) return CPB_OK;
    const int warps = 8;
    reparam_kernel<<<cdiv(batch, warps), warps * 32, 0, stream>>>(heads, eps, batch, zdim, pitch, kl_tolerance * zdim,
                                                                   kl_tolerance > 0.f ? 1 : 0, zout, kl_rows, kl_active);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_reparam_bwd(const float* heads, const float* eps, const float* gz, const float* kl_active,
                           int batch, int zdim, int pitch, float coef, float* gheads, cudaStream_t stream) {
    const long long n = (long long)batch * pitch;
    if (n == 0) return CPB_OK;
    reparam_bwd_kernel<<<cdiv(n, 256), 256, 0, stream>>>(heads, eps, gz, kl_active, batch, zdim, pitch, coef, gheads);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_pitch_copy(const float* src, int src_pitch, float* dst, int dst_pitch, int rows, cudaStream_t stream) {
    CPB_REQUIRE(src_pitch % 4 == 0 && dst_pitch % 4 == 0, "pitch_copy: pitches must be multiples of 4");
    const long long n4 = (long long)rows * (dst_pitch / 4);
    if (n4 == 0) return CPB_OK;
    pitch_copy_kernel<<<cdiv(n4, 256), 256, 0, stream>>>((const float4*)src, src_pitch / 4, (float4*)dst, dst_pitch / 4, n4);
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int LOSS>
static int32_t launch_recon_loss_t(const float* logits_p, const float* target_p, int batch, int npix, int ct, float gscale,
                                   float* frame_loss, float* dlogits_p, float* frame_dsum, cudaStream_t stream) {
    if (ct == 3)
        recon_loss_kernel<LOSS, 3><<<batch, 256, 0, stream>>>((const float4*)logits_p, (const float4*)target_p, npix,
                                                              gscale, frame_loss, (float4*)dlogits_p, frame_dsum);
    else
        recon_loss_kernel<LOSS, 1><<<batch, 256, 0, stream>>>((const float4*)logits_p, (const float4*)target_p, npix,
                                                              gscale, frame_loss, (float4*)dlogits_p, frame_dsum);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_recon_loss(const float* logits_p, const float* target_p, int batch, int npix, int ct, int loss_type,
                          float gscale, float* frame_loss, float* dlogits_p, cudaStream_t stream, float* frame_dsum) {
    CPB_REQUIRE(ct == 1 || ct == 3, "recon_loss: target_channels must be 1 or 3");
    if (batch == 0) return CPB_OK;
    switch (loss_type) {
        case CPB_LOSS_MSE: return launch_recon_loss_t<CPB_LOSS_MSE>(logits_p, target_p, batch, npix, ct, gscale, frame_loss, dlogits_p, frame_dsum, stream);
        case CPB_LOSS_BCE: return launch_recon_loss_t<CPB_LOSS_BCE>(logits_p, target_p, batch, npix, ct, gscale, frame_loss, dlogits_p, frame_dsum, stream);
        case CPB_LOSS_BCE_V2: return launch_recon_loss_t<CPB_LOSS_BCE_V2>(logits_p, target_p, batch, npix, ct, gscale, frame_loss, dlogits_p, frame_dsum, stream);
    }
    CPB_REQUIRE(false, "recon_loss: unknown loss_type %d", loss_type);
}

int32_t launch_prep_flat(const void* src, int dtype, float scale, long long n, float* dst, int32_t* flags, int flag_bit, cudaStream_t stream) {
    if (n == 0) return CPB_OK;
    const unsigned blocks = (unsigned)cdiv(n, 256);
    if (dtype == CPB_FRAME_F32) prep_flat_kernel<float><<<blocks, 256, 0, stream>>>((const float*)src, scale, n, dst, flags, flag_bit);
    else if (dtype == CPB_FRAME_U8) prep_flat_kernel<uint8_t><<<blocks, 256, 0, stream>>>((const uint8_t*)src, scale, n, dst, flags, flag_bit);
    else CPB_REQUIRE(false, "prep_flat: unknown frame dtype %d", dtype);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_sigmoid(const float* x, float* y, long long n, cudaStream_t stream) {
    if (n == 0) return CPB_OK;
    sigmoid_kernel<<<cdiv(n, 256), 256, 0, stream>>>(x, y, n);
    CPB_LAUNCHED();
    return CPB_OK;
}

// unpadded [B, n] logits / targets (n % 4 == 0): every float4 lane is a real element (the CT = 4 instantiation)
int32_t launch_recon_loss_flat(const float* logits, const float* target, int batch, int n, int loss_type, float gscale,
                               float* frame_loss, float* dlogits, cudaStream_t stream) {
    CPB_REQUIRE(n % 4 == 0, "recon_loss_flat: row length must be a multiple of 4");
    if (batch == 0) return CPB_OK;
    const int n4 = n / 4;
    switch (loss_type) {
        case CPB_LOSS_MSE: recon_loss_kernel<CPB_LOSS_MSE, 4><<<batch, 256, 0, stream>>>((const float4*)logits, (const float4*)target, n4, gscale, frame_loss, (float4*)dlogits, nullptr); break;
        case CPB_LOSS_BCE: recon_loss_kernel<CPB_LOSS_BCE, 4><<<batch, 256, 0, stream>>>((const float4*)logits, (const float4*)target, n4, gscale, frame_loss, (float4*)dlogits, nullptr); break;
        case CPB_LOSS_BCE_V2: recon_loss_kernel<CPB_LOSS_BCE_V2, 4><<<batch, 256, 0, stream>>>((const float4*)logits, (const float4*)target, n4, gscale, frame_loss, (float4*)dlogits, nullptr); break;
        default: CPB_REQUIRE(false, "recon_loss_flat: unknown loss_type %d", loss_type);
    }
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_finalize_losses(const float* frame_loss, const float* kl_rows, int batch, float scale,
                               float* losses, cudaStream_t stream) {
    finalize_losses_kernel<<<1, 1024, 0, stream>>>(frame_loss, kl_rows, batch, scale, losses);
    CPB_LAUNCHED();
    return CPB_OK;
}

long long colsum_scratch_floats(long long rows, int pitch) {
    return colsum_blocks(rows, pitch) * pitch;
}

int32_t launch_colsum(const float* g, long long rows, int pitch, int c_real, float* out, float* scratch,
                      cudaStream_t stream) {
    CPB_REQUIRE(pitch % 4 == 0, "colsum: pitch must be a multiple of 4");
    if (rows == 0) return CPB_OK;
    ProfScope prof("bias_grad.colsum", stream);
    const int nblocks = (int)colsum_blocks(rows, pitch);
    dim3 grid((unsigned)nblocks, (unsigned)cdiv(pitch >> 2, 256));
    colsum_kernel<<<grid, 256, 0, stream>>>(g, rows, pitch, scratch);
    CPB_LAUNCHED();
    colsum_final_kernel<<<cdiv(c_real, 8), 256, 0, stream>>>(scratch, nblocks, pitch, c_real, out);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_relayout(const float* params, float* dst, const RelayoutTable& table, cudaStream_t stream) {
    if (table.total == 0) return CPB_OK;
    relayout_kernel<<<cdiv(table.total, 256), 256, 0, stream>>>(params, dst, table);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_adam(float* params, const float* grads, float* m, float* v, long long n, float* powers,
                    float lr, const float* lr_dev, float beta1, float beta2, float epsilon, cudaStream_t stream,
                    const void* guard) {
    CPB_REQUIRE(n % 4 == 0, "adam: buffer length %lld is not a multiple of 4", n);
    if (n == 0) return CPB_OK;
    adam_kernel<<<cdiv(n / 4, 256), 256, 0, stream>>>((float4*)params, (const float4*)grads, (float4*)m, (float4*)v,
                                                      n / 4, powers, lr, lr_dev, beta1, beta2, epsilon, (const uint32_t*)guard);
    CPB_LAUNCHED();
    adam_powers_kernel<<<1, 1, 0, stream>>>(powers, beta1, beta2, (const uint32_t*)guard);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_fill_zero(float* p, long long n, cudaStream_t stream) {
    CPB_REQUIRE(n % 4 == 0, "fill_zero: length must be a multiple of 4");
    if (n == 0) return CPB_OK;
    fill_zero_kernel<<<cdiv(n / 4, 256), 256, 0, stream>>>((float4*)p, n / 4);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
