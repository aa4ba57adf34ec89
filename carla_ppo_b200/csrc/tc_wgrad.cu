// Tensor-core weight gradient for sm_90a (tf Conv2DBackpropFilter for conv and transposed-conv layers):
//
//   gw[i, j] = sum_{m}  big[row(m) + tap_off[i / run] + i % run] * small[m * J + j]        (same contract as wgrad.cu)
//
// as D[128 x BN] += A^T B with the REDUCTION index m on the MMA K axis.  In NHWC memory the channel index -- not m --
// is contiguous, while wgmma takes TF32 operands only K-major, so this kernel stages through registers: a loader thread
// reads the float4 of 4 channels at 4 consecutive reduction positions (4 x LDG.128), regroups them into 4 vectors
// "one channel x 4 positions" (4x4 register transpose), splits them into TF32 hi / lo parts and writes each as ONE
// 16-byte chunk of the K-major SWIZZLE_128B tile (8 STS.128).  A quarter-warp covers 8 consecutive channel groups of
// ONE position (a contiguous 128-byte line per LDG.128); the tile rows are permuted (channel 4*cg + c lives in row
// 32*c + cg) so that the swizzled stores stay conflict-free, and the accumulator rows / columns are un-permuted
// when the partial is stored.  Warps 0-7 load A and, as two warpgroups of 64 tile rows, issue the wgmma of the stage
// they just filled while the next k-block's loads are in flight; warps 8-11 load B; two k-blocks are in flight per
// loader thread; the position cursor advances without divisions.
// 3xTF32 products, the separate cross-term registers and the chunked accumulation into fp32 register accumulators are
// those of tc_tapgemm.cu.  Each (i-tile, j-tile, split) CTA of the single split-K wave writes its partial [128 x BN]
// block; reduce_partials() sums the splits in a fixed order (deterministic).
// Single-pass variant (PASSES = 1, math mode 2): the loaders round both operands to the nearest TF32 value and store
// the hi tiles only (a stage is A + B), one wgmma per 8-wide k-step into the chunk accumulator, no cross terms.
#include "tc_common.cuh"
#include "wgrad.cuh"

namespace cpb {

namespace {

using namespace tc;

constexpr int CHUNK_KB = 4;

template <int BN, int PASSES>
struct TcWgCfg {
    static constexpr int B_TILE_BYTES = BN * TBK * 4;
    static constexpr int PARTS = PASSES == 3 ? 2 : 1;                // tiles per operand: [hi | lo] or [hi]
    static constexpr int B_OFF = PARTS * A_TILE_BYTES;               // stage layout: A tile(s) | B tile(s)
    static constexpr int STAGE_BYTES = PARTS * A_TILE_BYTES + PARTS * B_TILE_BYTES;
    static constexpr int STAGES = (STAGE_BYTES * 4 <= 200 * 1024) ? 4 : 3;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
};

constexpr int kWgLoaderWarps = 8;                         // warps 0-7: A (big) loaders, wgmma, partial store
constexpr int kWgBWarps = 4;                              // warps 8-11: B (small) loaders
constexpr int kWgThreads = (kWgLoaderWarps + kWgBWarps) * 32;

template <int BN, int PASSES>
__global__ void __maxnreg__(168)     // 12 warps x 32 x 168 registers fit one SM
tc_wgrad_kernel(const __grid_constant__ WgradParams p) {
    static_assert(PASSES == 3 || PASSES == 1, "3xTF32 or a single TF32 pass");
    using Cfg = TcWgCfg<BN, PASSES>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int B_TILE_BYTES = Cfg::B_TILE_BYTES;
    constexpr int B_OFF = Cfg::B_OFF;
    constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;

    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES];     // loader warps -> wgmma (one arrival per warp)
    __shared__ uint64_t empty_bar[STAGES];    // wgmma warps -> loaders (one arrival per warp once its wgmma are done)

    const int tid = threadIdx.x;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform for the compiler
    const int i0 = blockIdx.x * TBM;
    const int j0 = blockIdx.y * BN;
    const int HoWo = p.Ho * p.Wo;
    const long long M = (long long)p.batch * HoWo;
    const long long m_begin = (long long)blockIdx.z * p.m_per_split;
    long long m_end = m_begin + p.m_per_split;
    if (m_end > M) m_end = M;
    // k-blocks of this split, rounded up to an even count: the loops below take two k-blocks per iteration (one per
    // register buffer) with no branch around the second, which ptxas would otherwise treat as divergent and answer by
    // serialising every wgmma (C7518).  The padding k-block loads nothing (positions >= len are zero-filled), and
    // adding zero products leaves the accumulators bit-for-bit unchanged.
    const int nkb = m_end > m_begin ? 2 * (int)((m_end - m_begin + 2 * TBK - 1) / (2 * TBK)) : 0;

    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], kWgLoaderWarps + kWgBWarps); mbar_init(&empty_bar[s], kWgLoaderWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    constexpr int BQ = BN / 4;                       // channel groups of the B tile
    const int len = (int)(m_end - m_begin);          // reduction positions of this split
    // 4x4 register transpose + split + store: x[j] = 4 channels at position j  ->  one chunk per channel
    // (single pass: rounded to nearest TF32, hi tile only)
    auto store_t = [&](uint32_t tile_hi, uint32_t tile_lo, const float4* x, const uint32_t* so) {
        const float xs[4][4] = {{x[0].x, x[1].x, x[2].x, x[3].x}, {x[0].y, x[1].y, x[2].y, x[3].y},
                                {x[0].z, x[1].z, x[2].z, x[3].z}, {x[0].w, x[1].w, x[2].w, x[3].w}};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if constexpr (PASSES == 3) {
                float4 hi, lo;
                split_tf32(xs[c][0], hi.x, lo.x); split_tf32(xs[c][1], hi.y, lo.y);
                split_tf32(xs[c][2], hi.z, lo.z); split_tf32(xs[c][3], hi.w, lo.w);
                asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(tile_hi + so[c]), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
                asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(tile_lo + so[c]), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
            } else {
                asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(tile_hi + so[c]), "r"(round_tf32(xs[c][0])),
                             "r"(round_tf32(xs[c][1])), "r"(round_tf32(xs[c][2])), "r"(round_tf32(xs[c][3])) : "memory");
            }
        }
    };

    if (warp >= kWgLoaderWarps) {
        // ================================ B (small) loaders ================================
        // 128 threads = (channel group of 4 output channels) x (position block of 4 reduction positions), a
        // quarter-warp again covering 128 contiguous bytes; BN = 32 leaves half of the threads idle.  Same 4x4
        // transpose + split + swizzled store as the A side.
        constexpr int NCGH = BQ >= 8 ? BQ / 8 : 1;
        const int r = (tid - kWgLoaderWarps * 32) >> 3;           // 0..15
        const int cgb = (r % NCGH) * 8 + (lane & 7);
        const int mb0 = r / NCGH;                                  // BN 32: 0..15 (>= 8 idle), 64: 0..7
        const bool active = mb0 < 8;
        uint32_t soffb[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int rb = BQ * c + cgb;
            soffb[c] = (uint32_t)((rb >> 3) * 1024 + (rb & 7) * 128 + ((mb0 ^ (rb & 7)) << 4));
        }
        int relB = mb0 * 4;
        const float* bptr = p.small + (m_begin + relB) * p.J + j0 + cgb * 4;
        auto load_b = [&](float4* xb) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                xb[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (active && relB + j < len) xb[j] = __ldg(reinterpret_cast<const float4*>(bptr + j * p.J));
            }
            relB += TBK;
            bptr += TBK * p.J;
        };
        float4 xb0[4], xb1[4];
        int sS = 0;
        uint32_t phS = 1;
        auto step_b = [&](int kb, float4* xb) {
            const uint32_t stage = smem_base + sS * STAGE_BYTES + B_OFF;
            mbar_wait(&empty_bar[sS], phS);
            if (active) store_t(stage, stage + B_TILE_BYTES, xb, soffb);
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[sS]);
            if (kb + 2 < nkb) load_b(xb);
            if (++sS == STAGES) { sS = 0; phS ^= 1u; }
        };
        if (nkb > 0) load_b(xb0);
        if (nkb > 1) load_b(xb1);
        for (int kb = 0; kb < nkb; kb += 2) {
            step_b(kb, xb0);
            step_b(kb + 1, xb1);
        }
    } else {
        // ================================ A loaders / wgmma / partial store ================================
        // thread = (channel group cg of 4 channels, position block mb of 4 reduction positions).
        // A quarter-warp = 8 consecutive channel groups of ONE position: its LDG.128 is one contiguous 128-byte line
        // (the L1 data pipe charges a wavefront per 32-byte sector when a quarter-warp straddles lines).
        // Conflict-free stores then need the 8 lanes to hit 8 different swizzle slots: channel 4*cg + c is kept in
        // tile row rho = 32*c + cg (A) / (BN/4)*c + cg (B), so a quarter-warp's rows differ in rho%8.  The
        // accumulator rows / columns come out permuted the same way and are un-permuted when the partial is stored.
        const int cg = (warp & 3) * 8 + (lane & 7);
        const int mb = (warp >> 2) * 4 + (lane >> 3);
        const int a_i = i0 + cg * 4;
        const bool a_col_ok = a_i < p.I;
        long long a_coloff = 0;
        if (a_col_ok) {
            const int tap = a_i / p.run;
            a_coloff = p.tap_off[tap] + (a_i - tap * p.run);
        }
        uint32_t soff[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int ra = 32 * c + cg;
            soff[c] = (uint32_t)((ra >> 3) * 1024 + (ra & 7) * 128 + ((mb ^ (ra & 7)) << 4));
        }

        // position cursor of this thread's NEXT load (k-block kbL): image n, position rem = oy*Wo + ox inside it.
        // Advancing by a k-block (32 positions) needs no division: oy comes from a multiply-high by ceil(2^32 / Wo).
        const uint32_t wo_magic = (uint32_t)((0x100000000ull + (uint32_t)p.Wo - 1) / (uint32_t)p.Wo);
        const int dx = p.sstride * p.big_pitch;                              // next position in the row
        const int drow = (p.sstride * p.Wb - p.Wo * p.sstride) * p.big_pitch;   // ... wrapping to the next row
        const int dimg = (int)(p.big_img - (long long)p.Ho * p.sstride * p.Wb * p.big_pitch);   // ... to the next image
        int nL, remL, relL = mb * 4;                               // relL: position index relative to m_begin
        {
            const long long m = m_begin + relL;
            nL = (int)(m / HoWo);
            remL = (int)(m - (long long)nL * HoWo);
        }
        auto load_regs = [&](float4* areg) {
            int oy = (int)__umulhi((uint32_t)remL, wo_magic);
            int ox = remL - oy * p.Wo;
            uint32_t off = (uint32_t)nL * (uint32_t)p.big_img + (uint32_t)((oy * p.sstride * p.Wb + ox * p.sstride) * p.big_pitch) + (uint32_t)a_coloff;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const bool v = relL + j < len;
                areg[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (v && a_col_ok) areg[j] = __ldg(reinterpret_cast<const float4*>(p.big + off));
                off += (uint32_t)dx;
                if (++ox == p.Wo) { ox = 0; off += (uint32_t)drow; if (++oy == p.Ho) { oy = 0; off += (uint32_t)dimg; } }
            }
            relL += TBK;
            remL += TBK;
            while (remL >= HoWo) { remL -= HoWo; ++nL; }
        };

        constexpr int HALF = BN / 2;                 // accumulator registers per thread for a 64 x BN product
        const int wg = warp >> 2;                    // warpgroup: tile rows [64*wg, 64*wg + 64)
        constexpr int DN = PASSES == 3 ? BN : HALF;
        float acc[HALF];                             // fp32 register accumulators (main + cross)
        float d[DN];                                 // chunk accumulators: [main (HALF) | cross (HALF, 3 passes only)]
#pragma unroll
        for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
#pragma unroll
        for (int i = 0; i < DN; ++i) d[i] = 0.f;

        // two k-blocks of operand rows are in flight per thread (register double buffer): with one, every
        // k-block costs a full L2 round trip per warp
        float4 xa0[4], xa1[4];
        int sS = 0;                                 // stage of the k-block being stored and the parity its empty
        uint32_t phS = 1;                           // barrier shows once free (fresh barrier: parity 1 counts as complete)
        int prev = -1;                              // stage whose wgmma group may still be in flight
        auto step = [&](int kb, float4* xa) {
            const int s = sS;
            const uint32_t stage = smem_base + s * STAGE_BYTES;
            mbar_wait(&empty_bar[s], phS);
            store_t(stage, stage + A_TILE_BYTES, xa, soff);
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[s]);
            if (kb + 2 < nkb) load_regs(xa);
            mbar_wait(&full_bar[s], (uint32_t)((kb / STAGES) & 1));
            const uint64_t a_hi = make_desc(stage + wg * (A_TILE_BYTES / 2));
            const uint64_t a_lo = make_desc(stage + A_TILE_BYTES + wg * (A_TILE_BYTES / 2));
            const uint64_t b_hi = make_desc(stage + B_OFF);
            const uint64_t b_lo = make_desc(stage + B_OFF + B_TILE_BYTES);
            // main (+)= a_hi x b_hi,  cross (+)= a_hi x b_lo,  cross += a_lo x b_hi (single pass: main (+)= a x b only).
            // Each product writes exactly one of the two disjoint accumulator arrays: a wgmma into a register range
            // that only partly overlaps an earlier one in flight (e.g. one N = 2*BN product over [main | cross]) makes
            // ptxas serialise the stream (C7511).
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < TBK / 8; ++ks) {
                const uint64_t adv = (uint64_t)(ks * 2);          // 32 bytes per k-step (K-major)
                const uint32_t keep = ((kb % CHUNK_KB) | ks) != 0 ? 1u : 0u;
                wgmma_tf32<BN>(d, a_hi + adv, b_hi + adv, keep);
                if constexpr (PASSES == 3) {
                    wgmma_tf32<BN>(d + HALF, a_hi + adv, b_lo + adv, keep);
                    wgmma_tf32<BN>(d + HALF, a_lo + adv, b_hi + adv, 1u);
                }
            }
            wgmma_commit();
            if (kb % CHUNK_KB == CHUNK_KB - 1 || kb == nkb - 1) {
                wgmma_wait<0>();
                fence_regs<DN>(d);
                if (lane == 0) {
                    if (prev >= 0) mbar_arrive(&empty_bar[prev]);
                    mbar_arrive(&empty_bar[s]);
                }
                prev = -1;
#pragma unroll
                for (int i = 0; i < HALF; ++i) {
                    acc[i] += d[i];
                    if constexpr (PASSES == 3) acc[i] += d[HALF + i];
                }
            } else {
                if (prev >= 0) {
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = s;
            }
            if (++sS == STAGES) { sS = 0; phS ^= 1u; }
        };
        if (nkb > 0) load_regs(xa0);
        if (nkb > 1) load_regs(xa1);
        for (int kb = 0; kb < nkb; kb += 2) {
            step(kb, xa0);
            step(kb + 1, xa1);
        }
        wgmma_wait<0>();     // a no-op (the last k-block ends a chunk); without it ptxas injects one before the stores

        // ---- partial[split][i][j]: tile row rho holds channel i = 4*(rho % 32) + rho / 32; accumulator column rb holds
        //      j = 4*(rb % BQ) + rb / BQ
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rho = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            const int i = i0 + 4 * (rho & 31) + (rho >> 5);
            if (i >= p.I) continue;
            float* out = p.partial + ((long long)blockIdx.z * p.I + i) * p.J + j0;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int rb = 8 * j + 2 * (lane & 3) + c;
                    out[4 * (rb % BQ) + rb / BQ] = acc[4 * j + 2 * h + c];
                }
        }
    }
}
template <int BN, int PASSES>
int32_t tc_wg_launch(const WgradParams& p, cudaStream_t stream) {
    dim3 grid((unsigned)cdiv(p.I, TBM), (unsigned)(p.J / BN), (unsigned)p.splits);
    tc_wgrad_kernel<BN, PASSES><<<grid, kWgThreads, TcWgCfg<BN, PASSES>::SMEM_BYTES, stream>>>(p);
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int BN, int PASSES>
int32_t tc_wg_init_one() {
    CPB_CUDA(cudaFuncSetAttribute(tc_wgrad_kernel<BN, PASSES>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcWgCfg<BN, PASSES>::SMEM_BYTES));
    return CPB_OK;
}

int tc_wg_bn(int J) { return J % 64 == 0 ? 64 : 32; }   // at most 64: see tc_bn

}  // namespace

int32_t tc_wgrad_init() {
    CPB_TRY((tc_wg_init_one<32, 3>()));
    CPB_TRY((tc_wg_init_one<64, 3>()));
    CPB_TRY((tc_wg_init_one<32, 1>()));
    CPB_TRY((tc_wg_init_one<64, 1>()));
    return CPB_OK;
}

bool tc_wgrad_supported(int I, int J, int run) { return run % 4 == 0 && J % 32 == 0 && I >= 128; }

int tc_wgrad_pick_splits(int I, int J, long long M) {
    const long long tiles = (long long)cdiv(I, TBM) * (J / tc_wg_bn(J));
    long long splits = kTcWaveCtas / tiles;                 // ONE wave: one CTA per SM (193 KB of shared memory each)
    const long long max_splits = (M + 1023) / 1024;         // keep >= 1024 reduction positions per split
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    return (int)splits;
}

int32_t launch_tc_wgrad(const WgradParams& p, cudaStream_t stream) {
    CPB_REQUIRE(tc_wgrad_supported(p.I, p.J, p.run) && p.I == p.ntaps * p.run, "tc_wgrad: unsupported problem (I=%d J=%d)", p.I, p.J);
    CPB_REQUIRE(p.m_per_split % TBK == 0 && p.splits >= 1, "tc_wgrad: bad split");
    CPB_REQUIRE((long long)p.batch * p.big_img < (1ll << 31) && p.m_per_split < (1ll << 30) && p.Wo < 65536 && p.Ho * p.Wo < 65536,
                "tc_wgrad: tensor too large for 32-bit offsets");
    CPB_REQUIRE(p.passes == 3 || p.passes == 1, "tc_wgrad: passes must be 3 or 1, got %d", p.passes);
    if (p.passes == 1) return tc_wg_bn(p.J) == 64 ? tc_wg_launch<64, 1>(p, stream) : tc_wg_launch<32, 1>(p, stream);
    return tc_wg_bn(p.J) == 64 ? tc_wg_launch<64, 3>(p, stream) : tc_wg_launch<32, 3>(p, stream);
}

}  // namespace cpb
