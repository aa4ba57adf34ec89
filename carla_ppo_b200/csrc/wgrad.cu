// fp32 SIMT weight-gradient GEMM with split reduction (see wgrad.cuh).
#include "wgrad.cuh"

namespace cpb {

namespace {

constexpr int BKM = 16;   // reduction positions per pipeline stage

template <int BI, int BJ, int TI, int TJ, int STAGES, int MINB>
__global__ void __launch_bounds__((BI / TI) * (BJ / TJ), MINB)
wgrad_kernel(const __grid_constant__ WgradParams p) {
    constexpr int NT = (BI / TI) * (BJ / TJ);
    constexpr int TXJ = BJ / TJ;
    constexpr int GI = TI / 4, GJ = TJ / 4;
    constexpr int ISTEP = BI / GI, JSTEP = BJ / GJ;
    constexpr int A_F4 = BKM * BI / 4, B_F4 = BKM * BJ / 4;
    constexpr int A_ITERS = (A_F4 + NT - 1) / NT, B_ITERS = (B_F4 + NT - 1) / NT;
    static_assert(NT % (BI / 4) == 0 && NT % (BJ / 4) == 0, "loader columns must be thread-invariant");

    extern __shared__ __align__(16) float smem[];
    float* As = smem;                        // [STAGES][BKM][BI]
    float* Bs = smem + STAGES * BKM * BI;    // [STAGES][BKM][BJ]

    const int tid = threadIdx.x;
    const int tj = tid % TXJ;
    const int ti = tid / TXJ;
    const int i0 = blockIdx.x * BI;
    const int j0 = blockIdx.y * BJ;
    const int HoWo = p.Ho * p.Wo;
    const long long M = (long long)p.batch * HoWo;
    const long long m_begin = (long long)blockIdx.z * p.m_per_split;
    long long m_end = m_begin + p.m_per_split;
    if (m_end > M) m_end = M;

    // loader column of this thread inside the A tile (constant over the loop)
    const int a_col = (tid % (BI / 4)) * 4;
    const int a_i = i0 + a_col;
    const bool a_col_ok = a_i < p.I;
    long long a_coloff = 0;
    if (a_col_ok) {
        const int tap = a_i / p.run;
        a_coloff = p.tap_off[tap] + (a_i - tap * p.run);
    }
    const int b_col = (tid % (BJ / 4)) * 4;

    auto load_stage = [&](int stage, long long mb) {
        float* as = As + stage * BKM * BI;
#pragma unroll
        for (int it = 0; it < A_ITERS; ++it) {
            const int f = tid + it * NT;
            if (A_F4 % NT == 0 || f < A_F4) {
                const int mm = f / (BI / 4);
                const long long m = mb + mm;
                const bool v = a_col_ok && m < m_end;
                const float* g = p.big;
                if (v) {
                    const int n = (int)(m / HoWo);
                    const int rem = (int)(m - (long long)n * HoWo);
                    const int oy = rem / p.Wo;
                    const int ox = rem - oy * p.Wo;
                    g = p.big + (long long)n * p.big_img +
                        ((long long)(oy * p.sstride) * p.Wb + ox * p.sstride) * p.big_pitch + a_coloff;
                }
                cp_async16(as + mm * BI + a_col, g, v);
            }
        }
        float* bs = Bs + stage * BKM * BJ;
#pragma unroll
        for (int it = 0; it < B_ITERS; ++it) {
            const int f = tid + it * NT;
            if (B_F4 % NT == 0 || f < B_F4) {
                const int mm = f / (BJ / 4);
                const long long m = mb + mm;
                const bool v = m < m_end;
                const float* g = v ? p.small + m * p.J + j0 + b_col : p.small;
                cp_async16(bs + mm * BJ + b_col, g, v);
            }
        }
    };

    float acc[TI][TJ];
#pragma unroll
    for (int i = 0; i < TI; ++i)
#pragma unroll
        for (int j = 0; j < TJ; ++j) acc[i][j] = 0.f;

    const int nkb = m_end > m_begin ? (int)((m_end - m_begin + BKM - 1) / BKM) : 0;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nkb) load_stage(s, m_begin + (long long)s * BKM);
        cp_async_commit();
    }
    for (int kb = 0; kb < nkb; ++kb) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        const int nxt = kb + STAGES - 1;
        if (nxt < nkb) load_stage(nxt % STAGES, m_begin + (long long)nxt * BKM);
        cp_async_commit();
        const float* as = As + (kb % STAGES) * BKM * BI + ti * 4;
        const float* bs = Bs + (kb % STAGES) * BKM * BJ + tj * 4;
#pragma unroll
        for (int mm = 0; mm < BKM; ++mm) {
            float a[TI], b[TJ];
#pragma unroll
            for (int g = 0; g < GI; ++g) {
                const float4 t = *reinterpret_cast<const float4*>(as + mm * BI + g * ISTEP);
                a[g * 4 + 0] = t.x; a[g * 4 + 1] = t.y; a[g * 4 + 2] = t.z; a[g * 4 + 3] = t.w;
            }
#pragma unroll
            for (int g = 0; g < GJ; ++g) {
                const float4 t = *reinterpret_cast<const float4*>(bs + mm * BJ + g * JSTEP);
                b[g * 4 + 0] = t.x; b[g * 4 + 1] = t.y; b[g * 4 + 2] = t.z; b[g * 4 + 3] = t.w;
            }
#pragma unroll
            for (int i = 0; i < TI; ++i)
#pragma unroll
                for (int j = 0; j < TJ; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
    }
    cp_async_wait<0>();

    float* out = p.partial + (long long)blockIdx.z * p.I * p.J;
#pragma unroll
    for (int gi = 0; gi < GI; ++gi)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int i = i0 + ti * 4 + gi * ISTEP + q;
            if (i >= p.I) continue;
#pragma unroll
            for (int gj = 0; gj < GJ; ++gj) {
                float4 v;
                v.x = acc[gi * 4 + q][gj * 4 + 0]; v.y = acc[gi * 4 + q][gj * 4 + 1];
                v.z = acc[gi * 4 + q][gj * 4 + 2]; v.w = acc[gi * 4 + q][gj * 4 + 3];
                *reinterpret_cast<float4*>(out + (long long)i * p.J + j0 + tj * 4 + gj * JSTEP) = v;
            }
        }
}

template <int BI, int BJ, int TI, int TJ, int STAGES, int MINB>
int32_t launch_cfg(const WgradParams& p, cudaStream_t stream) {
    constexpr int NT = (BI / TI) * (BJ / TJ);
    constexpr int smem = STAGES * BKM * (BI + BJ) * (int)sizeof(float);
    dim3 grid((unsigned)cdiv(p.I, BI), (unsigned)(p.J / BJ), (unsigned)p.splits);
    wgrad_kernel<BI, BJ, TI, TJ, STAGES, MINB><<<grid, NT, smem, stream>>>(p);
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int BI, int BJ, int TI, int TJ, int STAGES, int MINB>
int32_t init_cfg() {
    constexpr int smem = STAGES * BKM * (BI + BJ) * (int)sizeof(float);
    CPB_CUDA(cudaFuncSetAttribute(wgrad_kernel<BI, BJ, TI, TJ, STAGES, MINB>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return CPB_OK;
}

#define CPB_WG_A 128, 128, 8, 8, 3, 2
#define CPB_WG_B 128, 64, 8, 4, 3, 2
#define CPB_WG_C 64, 128, 4, 8, 3, 2
#define CPB_WG_D 64, 32, 4, 4, 4, 4

// 0..3 = A..D
int pick_tile(int I, int J) {
    if (J % 128 == 0) return I >= 128 ? 0 : 2;
    if (J % 64 == 0) return 1;
    return 3;
}
void tile_dims(int tile, int& bi, int& bj) {
    static const int dims[4][2] = {{128, 128}, {128, 64}, {64, 128}, {64, 32}};
    bi = dims[tile][0];
    bj = dims[tile][1];
}

// block = 32 outputs x 8 split-lanes; each lane sums splits l, l+8, ... and the 8 lane sums are
// combined in a fixed order (deterministic).
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ partial, int splits, long long IJ, int J, int c_pad, int c_real,
                       int j_real, float* __restrict__ out) {
    __shared__ float red[8][33];
    const int o = threadIdx.x & 31;
    const int l = threadIdx.x >> 5;
    const long long idx = (long long)blockIdx.x * 32 + o;
    float s = 0.f;
    if (idx < IJ)
        for (int k = l; k < splits; k += 8) s += partial[(long long)k * IJ + idx];
    red[l][o] = s;
    __syncthreads();
    if (l != 0 || idx >= IJ) return;
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) tot += red[k][o];
    const int j = (int)(idx % J);
    const int i = (int)(idx / J);
    const int t = i / c_pad;
    const int c = i - t * c_pad;
    if (c >= c_real || j >= j_real) return;
    out[((long long)t * c_real + c) * j_real + j] = tot;
}

// out[j][i] = sum_s partial[s][i][j] (splits in order) through a 32 x 32 shared-memory tile: reads and writes coalesced
__global__ void __launch_bounds__(256)
reduce_partials_t_kernel(const float* __restrict__ partial, int splits, int I, int J, float* __restrict__ out) {
    __shared__ float tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
    const long long IJ = (long long)I * J;
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const long long at = (long long)(i0 + r) * J + j0 + tx;
        float s = 0.f;
        for (int k = 0; k < splits; ++k) s += partial[(long long)k * IJ + at];
        tile[r][tx] = s;
    }
    __syncthreads();
#pragma unroll
    for (int r = ty; r < 32; r += 8) out[(long long)(j0 + r) * I + i0 + tx] = tile[tx][r];
}

}  // namespace

int32_t launch_reduce_partials_t(const float* partial, int splits, int I, int J, float* out, cudaStream_t stream) {
    CPB_REQUIRE(I % 32 == 0 && J % 32 == 0 && splits >= 1, "reduce_partials_t: I=%d, J=%d must be multiples of 32", I, J);
    reduce_partials_t_kernel<<<dim3((unsigned)(I / 32), (unsigned)(J / 32)), 256, 0, stream>>>(partial, splits, I, J, out);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t wgrad_init() {
    CPB_TRY((init_cfg<CPB_WG_A>()));
    CPB_TRY((init_cfg<CPB_WG_B>()));
    CPB_TRY((init_cfg<CPB_WG_C>()));
    CPB_TRY((init_cfg<CPB_WG_D>()));
    return CPB_OK;
}

int wgrad_pick_splits(int I, int J, long long M) {
    int bi, bj;
    tile_dims(pick_tile(I, J), bi, bj);
    const long long tiles = (long long)cdiv(I, bi) * (J / bj);
    long long target = 132 * 4;                   // ~2 waves at 2 CTAs/SM (132 SMs)
    long long splits = (target + tiles - 1) / tiles;
    const long long max_splits = (M + 255) / 256;  // keep >= 256 reduction positions per split
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    return (int)splits;
}

int32_t launch_wgrad(const WgradParams& p, cudaStream_t stream) {
    CPB_REQUIRE(p.run % 4 == 0 && p.I == p.ntaps * p.run, "wgrad: bad run/taps (I=%d, ntaps=%d, run=%d)", p.I, p.ntaps, p.run);
    CPB_REQUIRE(p.J % 32 == 0, "wgrad: J=%d is not a multiple of 32", p.J);
    CPB_REQUIRE(p.m_per_split % BKM == 0 && p.splits >= 1, "wgrad: bad split");
    switch (pick_tile(p.I, p.J)) {
        case 0: return launch_cfg<CPB_WG_A>(p, stream);
        case 1: return launch_cfg<CPB_WG_B>(p, stream);
        case 2: return launch_cfg<CPB_WG_C>(p, stream);
        default: return launch_cfg<CPB_WG_D>(p, stream);
    }
}

int32_t launch_reduce_partials(const float* partial, int splits, int I, int J, int c_pad, int c_real, int j_real,
                               float* out, cudaStream_t stream) {
    const long long IJ = (long long)I * J;
    reduce_partials_kernel<<<cdiv(IJ, 32), 256, 0, stream>>>(partial, splits, IJ, J, c_pad, c_real, j_real, out);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
