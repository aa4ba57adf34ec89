// fp32 SIMT tap-GEMM (see tapgemm.cuh).  cp.async multi-stage pipeline into padded shared
// memory, TMxTN register micro-tiles, float4 shared loads on both operands, fused
// bias / ReLU / ReLU-mask epilogue with float4 stores.
#include "tapgemm.cuh"

namespace cpb {

namespace {

constexpr int BK = 16;
constexpr int LDA = BK + 4;   // padded A row (floats): float4-aligned, conflict-free across rows

template <int BM, int BN, int TM, int TN, int STAGES>
struct TileCfg {
    static constexpr int kThreads = (BM / TM) * (BN / TN);
    static constexpr int kSmemBytes = STAGES * (BM * LDA + BK * BN) * (int)sizeof(float);
};

template <int BM, int BN, int TM, int TN, int STAGES, int MINB>
__global__ void __launch_bounds__((BM / TM) * (BN / TN), MINB)
tapgemm_kernel(const __grid_constant__ TapGemmParams p) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int TXN = BN / TN;               // threads along n
    constexpr int RSTEP = BM / TM;             // row interleave of a thread's micro-tile
    constexpr int G = TN / 4;                  // float4 column groups per thread
    constexpr int CSTEP = BN / G;              // column distance between groups
    constexpr int A_ITERS = (BM * (BK / 4) + NT - 1) / NT;
    constexpr int B_F4 = BK * BN / 4;
    constexpr int B_ITERS = (B_F4 + NT - 1) / NT;
    static_assert(BM * (BK / 4) % NT == 0, "A tile must divide evenly");

    extern __shared__ __align__(16) float smem[];
    float* As = smem;
    float* Bs = smem + STAGES * BM * LDA;

    const int tid = threadIdx.x;
    const int tx = tid % TXN;
    const int ty = tid / TXN;
    const int cls_id = blockIdx.z % p.nclass;
    const int yb = (blockIdx.z / p.nclass) % p.ybatch;
    const int ks = blockIdx.z / (p.nclass * p.ybatch);          // k-split index (ksplit > 1: dense layers with few rows)
    const TapClass& cls = p.cls[cls_id];
    const int Wo = cls.Wo;
    const int HoWo = cls.Ho * Wo;
    const long long M = (long long)p.batch * HoWo;
    const long long m0 = (long long)blockIdx.x * BM;
    if (m0 >= M) return;
    const int n0 = blockIdx.y * BN;
    const float* wsrc = p.wmat + yb * p.w_ystride + n0;

    // ---- per-thread A-loader rows (fixed for the whole k loop)
    const int a_kq = tid & 3;
    long long a_base[A_ITERS];
    int a_iy[A_ITERS], a_ix[A_ITERS];
    bool a_ok[A_ITERS];
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) {
        const int r = (tid >> 2) + i * (NT / 4);
        const long long m = m0 + r;
        a_ok[i] = m < M;
        const long long mm = a_ok[i] ? m : 0;
        const int n = (int)(mm / HoWo);
        const int rem = (int)(mm - (long long)n * HoWo);
        const int oy = rem / Wo;
        const int ox = rem - oy * Wo;
        a_iy[i] = oy * p.sstride;
        a_ix[i] = ox * p.sstride;
        a_base[i] = (long long)n * p.src_img + ((long long)a_iy[i] * p.Ws + a_ix[i]) * p.src_pitch + a_kq * 4;
    }

    auto load_stage = [&](int stage, int tap_idx, int c0) {
        const Tap& t = cls.taps[tap_idx];
        float* as = As + stage * BM * LDA;
#pragma unroll
        for (int i = 0; i < A_ITERS; ++i) {
            const int r = (tid >> 2) + i * (NT / 4);
            bool v = a_ok[i];
            if (p.check) {
                v = v && (unsigned)(a_iy[i] + t.dy) < (unsigned)p.Hs && (unsigned)(a_ix[i] + t.dx) < (unsigned)p.Ws;
            }
            const float* g = v ? p.src + a_base[i] + t.src_off + c0 : p.src;
            cp_async16(as + r * LDA + a_kq * 4, g, v);
        }
        float* bs = Bs + stage * BK * BN;
        const float* wt = wsrc + t.w_off + (long long)c0 * p.ldw;
#pragma unroll
        for (int i = 0; i < B_ITERS; ++i) {
            const int f = tid + i * NT;
            if (B_F4 % NT == 0 || f < B_F4) {
                const int k = f / (BN / 4);
                const int c4 = f % (BN / 4);
                cp_async16(bs + k * BN + c4 * 4, wt + (long long)k * p.ldw + c4 * 4, true);
            }
        }
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    // this CTA's share of the k-blocks (all of them unless the problem is k-split)
    const int nkb_all = cls.ntaps * (p.C / BK);
    const int kb_begin = (int)((long long)nkb_all * ks / p.ksplit);
    const int nkb = (int)((long long)nkb_all * (ks + 1) / p.ksplit) - kb_begin;
    int ld_tap = kb_begin / (p.C / BK), ld_c = (kb_begin % (p.C / BK)) * BK;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nkb) {
            load_stage(s, ld_tap, ld_c);
            ld_c += BK;
            if (ld_c == p.C) { ld_c = 0; ++ld_tap; }
        }
        cp_async_commit();
    }

    for (int kb = 0; kb < nkb; ++kb) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        const int nxt = kb + STAGES - 1;
        if (nxt < nkb) {
            load_stage(nxt % STAGES, ld_tap, ld_c);
            ld_c += BK;
            if (ld_c == p.C) { ld_c = 0; ++ld_tap; }
        }
        cp_async_commit();

        const float* as = As + (kb % STAGES) * BM * LDA + ty * LDA;
        const float* bs = Bs + (kb % STAGES) * BK * BN + tx * 4;
#pragma unroll
        for (int k4 = 0; k4 < BK / 4; ++k4) {
            float4 av[TM];
#pragma unroll
            for (int i = 0; i < TM; ++i) av[i] = *reinterpret_cast<const float4*>(as + i * RSTEP * LDA + k4 * 4);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                float bv[TN];
#pragma unroll
                for (int g = 0; g < G; ++g) {
                    const float4 t = *reinterpret_cast<const float4*>(bs + (k4 * 4 + kk) * BN + g * CSTEP);
                    bv[g * 4 + 0] = t.x; bv[g * 4 + 1] = t.y; bv[g * 4 + 2] = t.z; bv[g * 4 + 3] = t.w;
                }
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    const float a = kk == 0 ? av[i].x : kk == 1 ? av[i].y : kk == 2 ? av[i].z : av[i].w;
#pragma unroll
                    for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a, bv[j], acc[i][j]);
                }
            }
        }
    }
    cp_async_wait<0>();

    // ---- epilogue
    float bvals[TN];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int q = 0; q < 4; ++q)
            bvals[g * 4 + q] = p.bias ? p.bias[yb * p.bias_ystride + n0 + tx * 4 + g * CSTEP + q] : 0.f;

    float* dst = p.dst + yb * p.dst_ystride;
    const bool partial_out = p.ksplit > 1;                      // raw sums; ksplit_reduce adds bias / ReLU
    if (partial_out) dst = p.kpartial + (long long)ks * p.kpartial_stride + yb * p.dst_ystride;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const long long m = m0 + ty + i * RSTEP;
        if (m >= M) continue;
        const int n = (int)(m / HoWo);
        const int rem = (int)(m - (long long)n * HoWo);
        const int oy = rem / Wo;
        const int ox = rem - oy * Wo;
        const long long off = (long long)n * p.dst_img +
                              ((long long)(oy * p.dstride + cls.py) * p.Wd + (ox * p.dstride + cls.px)) * p.dst_pitch +
                              n0 + tx * 4;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            float4 v;
            if (partial_out) {
                *reinterpret_cast<float4*>(dst + off + g * CSTEP) =
                    make_float4(acc[i][g * 4 + 0], acc[i][g * 4 + 1], acc[i][g * 4 + 2], acc[i][g * 4 + 3]);
                continue;
            }
            v.x = acc[i][g * 4 + 0] + bvals[g * 4 + 0];
            v.y = acc[i][g * 4 + 1] + bvals[g * 4 + 1];
            v.z = acc[i][g * 4 + 2] + bvals[g * 4 + 2];
            v.w = acc[i][g * 4 + 3] + bvals[g * 4 + 3];
            if (p.relu) {
                v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
            }
            if (p.mask) {
                const float4 mk = *reinterpret_cast<const float4*>(p.mask + off + g * CSTEP);
                v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f;
                v.z = mk.z > 0.f ? v.z : 0.f; v.w = mk.w > 0.f ? v.w : 0.f;
            }
            *reinterpret_cast<float4*>(dst + off + g * CSTEP) = v;
        }
    }
}

template <int BM, int BN, int TM, int TN, int STAGES, int MINB>
int32_t launch_cfg(const TapGemmParams& p, cudaStream_t stream) {
    using Cfg = TileCfg<BM, BN, TM, TN, STAGES>;
    long long max_m = 0;
    for (int c = 0; c < p.nclass; ++c) {
        long long m = (long long)p.batch * p.cls[c].Ho * p.cls[c].Wo;
        if (m > max_m) max_m = m;
    }
    if (max_m == 0) return CPB_OK;
    dim3 grid((unsigned)((max_m + BM - 1) / BM), (unsigned)(p.N / BN), (unsigned)(p.nclass * p.ybatch * p.ksplit));
    tapgemm_kernel<BM, BN, TM, TN, STAGES, MINB><<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(p);
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int BM, int BN, int TM, int TN, int STAGES, int MINB>
int32_t init_cfg() {
    using Cfg = TileCfg<BM, BN, TM, TN, STAGES>;
    CPB_CUDA(cudaFuncSetAttribute(tapgemm_kernel<BM, BN, TM, TN, STAGES, MINB>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    return CPB_OK;
}

// out[e] = epilogue( sum_s partial[s][e] ) for the k-split dense problems: e runs over [ybatch][rows][N]; the mask
// (ybatch == 1 only) has the shape of dst
__global__ void ksplit_reduce_kernel(const float* __restrict__ partial, long long stride, int ksplit, long long total,
                                     int N, long long ystride, const float* __restrict__ bias, long long bias_ystride,
                                     int relu, const float* __restrict__ mask, float* __restrict__ dst) {
    const long long e4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e4 * 4 >= total) return;
    const long long e = e4 * 4;
    float4 a = *reinterpret_cast<const float4*>(partial + e);
    for (int s = 1; s < ksplit; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(partial + (long long)s * stride + e);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    if (bias != nullptr) {
        const long long yb = ystride > 0 ? e / ystride : 0;
        const int col = (int)((e - yb * ystride) % N);
        const float4 b = *reinterpret_cast<const float4*>(bias + yb * bias_ystride + col);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    if (relu) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
    if (mask != nullptr) {
        const float4 mk = *reinterpret_cast<const float4*>(mask + e);
        a.x = mk.x > 0.f ? a.x : 0.f; a.y = mk.y > 0.f ? a.y : 0.f; a.z = mk.z > 0.f ? a.z : 0.f; a.w = mk.w > 0.f ? a.w : 0.f;
    }
    *reinterpret_cast<float4*>(dst + e) = a;
}

}  // namespace

#define CPB_TILE_A 128, 128, 8, 8, 3, 2
#define CPB_TILE_B 256, 64, 8, 8, 3, 1
#define CPB_TILE_C 256, 32, 8, 4, 3, 1
#define CPB_TILE_D 64, 64, 4, 4, 4, 2

int32_t tapgemm_init() {
    CPB_TRY((init_cfg<CPB_TILE_A>()));
    CPB_TRY((init_cfg<CPB_TILE_B>()));
    CPB_TRY((init_cfg<CPB_TILE_C>()));
    CPB_TRY((init_cfg<CPB_TILE_D>()));
    return CPB_OK;
}

int32_t launch_tapgemm(const TapGemmParams& p, cudaStream_t stream) {
    CPB_REQUIRE(p.C % BK == 0 && p.C > 0, "tapgemm: C=%d is not a positive multiple of %d", p.C, BK);
    CPB_REQUIRE(p.N % 32 == 0 && p.N > 0, "tapgemm: N=%d is not a positive multiple of 32", p.N);
    CPB_REQUIRE(p.nclass == 1 || p.nclass == 4, "tapgemm: nclass must be 1 or 4");
    CPB_REQUIRE(p.ybatch >= 1, "tapgemm: ybatch must be >= 1");
    long long max_m = 0;
    for (int c = 0; c < p.nclass; ++c) {
        CPB_REQUIRE(p.cls[c].ntaps >= 1 && p.cls[c].ntaps <= kMaxTaps, "tapgemm: bad tap count");
        long long m = (long long)p.batch * p.cls[c].Ho * p.cls[c].Wo;
        if (m > max_m) max_m = m;
    }
    CPB_REQUIRE(p.ksplit >= 1 && p.ksplit <= kMaxKSplit, "tapgemm: bad ksplit");
    if (p.ksplit > 1) {
        // dense layers with few rows and a long reduction (heads fwd, dense1 dgrad: K = 6144): a handful of CTAs
        // walking 384 k-blocks each is latency bound at any batch size; split the reduction over gridDim.z
        CPB_REQUIRE(p.nclass == 1 && p.cls[0].Ho == 1 && p.cls[0].Wo == 1 && p.mask == nullptr && p.kpartial != nullptr &&
                    p.dst_pitch == p.N && p.N % 64 == 0, "tapgemm: k-split only for dense layers");
        CPB_TRY((launch_cfg<CPB_TILE_D>(p, stream)));
        return launch_ksplit_reduce(p, stream);
    }
    if (p.N % 128 == 0) return launch_cfg<CPB_TILE_A>(p, stream);
    if (p.N % 64 == 0) {
        if (max_m <= 16384) return launch_cfg<CPB_TILE_D>(p, stream);
        return launch_cfg<CPB_TILE_B>(p, stream);
    }
    return launch_cfg<CPB_TILE_C>(p, stream);
}

int32_t launch_ksplit_reduce(const TapGemmParams& p, cudaStream_t stream) {
    CPB_REQUIRE(p.mask == nullptr || p.ybatch == 1, "ksplit_reduce: a ReLU mask needs ybatch == 1");
    const long long total = p.ybatch > 1 ? (long long)p.ybatch * p.dst_ystride : (long long)p.batch * p.N;
    ksplit_reduce_kernel<<<cdiv(total / 4, 256), 256, 0, stream>>>(p.kpartial, p.kpartial_stride, p.ksplit, total, p.N,
                                                                 p.ybatch > 1 ? p.dst_ystride : 0, p.bias, p.bias_ystride,
                                                                 p.relu, p.mask, p.dst);
    CPB_LAUNCHED();
    return CPB_OK;
}

int tapgemm_pick_ksplit(int rows, int N, int ybatch, int K) {
    // A function of K ONLY: the arithmetic a frame sees must not depend on the batch it is in (the B=4096 property
    // test compares a batch with its quarters; a 1-ulp difference in the heads flips ReLUs downstream).
    (void)rows; (void)N; (void)ybatch;
    int s = kMaxKSplit;
    while (s > 1 && (K / 16) / s < 24) --s;                     // keep >= 24 k-blocks per CTA
    return s;
}

}  // namespace cpb
