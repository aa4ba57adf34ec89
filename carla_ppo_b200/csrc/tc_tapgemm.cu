// Tensor-core tap-GEMM for sm_90a: the same contraction as tapgemm.cu, computed with wgmma.mma_async
// (kind tf32, fp32 accumulators in registers) using the error-compensated 3xTF32 split
//
//     a*b  ~=  a_hi*b_hi + a_lo*b_hi + a_hi*b_lo ,   x_hi = x with the 13 low mantissa bits cleared,  x_lo = x - x_hi
//
// so that results stay fp32-accurate (relative error ~1e-6; a single TF32 pass gives ~3e-4 and would break the
// 1e-5 parity bar).  The tensor core itself ignores the 13 low mantissa bits of a TF32 operand, so the raw fp32
// tensor IS x_hi; x_lo is a second fp32 plane (written by the producing kernel's epilogue, or by lo_plane_kernel).
// Operands are staged in shared memory in the wgmma canonical K-major SWIZZLE_128B layout (rows of 32 floats =
// 128 B, 8-row groups of 1024 B, 16-byte chunk index XOR row%8) -- the only layout wgmma accepts for TF32 operands:
//   * A (activations, gathered rows) : cp.async 16 B per thread and row from the raw tensor (hi) and its lo plane,
//                                      zero-filled outside the image, completion counted on the stage's mbarrier;
//   * B (weights)                    : stored by tc_weights_kernel as ready-made swizzled tile images [hi | lo]; one
//                                      cp.async.bulk per k-block (multicast to the CTAs of a cluster).
// Persistent, warp-specialised kernel (see tc_tapgemm_kernel): two consumer warpgroups (64 tile rows each, 8 wgmma per
// 32-wide k-block: [main | cross] (+)= a_hi x [b_hi | b_lo] with N = 2*BN, cross += a_lo x b_hi) and four A-loader warps,
// the first lane of which also issues the weight-tile copies.
//
// Accumulation.  The tensor core adds into its fp32 accumulator with truncation, which shrinks a long running sum
// systematically (relative bias growing linearly with K).  Two measures bring this back to fp32-FMA level:
//   * the cross terms (2^-11 of the main term) accumulate in their OWN registers, so they do not re-truncate the
//     large accumulator;
//   * wgmma accumulation only runs over chunks of 128 k (4 k-blocks); each finished chunk is added to per-thread fp32
//     register accumulators (round-to-nearest).
// The register accumulators feed the bias / ReLU / ReLU-mask epilogue directly; the epilogue also writes the lo plane
// of its output when the consumer is another tensor-core layer.
#include "tapgemm.cuh"
#include "tc_common.cuh"

namespace cpb {

namespace {

using namespace tc;

template <int BN>
struct TcCfg {
    static constexpr int B_TILE_BYTES = BN * TBK * 4;
    static constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
    static constexpr int STAGES = (STAGE_BYTES * 4 <= 200 * 1024) ? 4 : 3;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;   // +1024: manual 1 KB alignment
};
constexpr int CHUNK_KB = 4;   // k-blocks accumulated by the tensor core before adding into the fp32 register accumulators

constexpr int kConsumerWarps = 8;                     // warps 0-7: two wgmma warpgroups + epilogue
constexpr int kLoaderWarp0 = 8;                       // warps 8-11: A loaders (cp.async)
constexpr int kLoaderWarps = 4;
constexpr int kLoaderThreads = kLoaderWarps * 32;
constexpr int kTcThreads = 384;                       // a multiple of 4 warps: registers are granted per 4 warps

int g_tc_cluster = 1;         // CTAs per cluster = multicast width of the weight tiles (CPB_TC_CLUSTER, 1/2/4/8)
int g_tc_clusters[2] = {0, 0};   // co-resident clusters of the persistent grid, per BN instantiation (32/64)

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_count_x() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy (TMA engine, no tensor map), completion counted in bytes on an mbarrier; with a CTA
// mask the same bytes land at the same shared offsets (data and barrier) of every CTA of the cluster in the mask
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask, bool multicast) {
    if (multicast)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                     ::"r"(dst), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask) : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// PERSISTENT, CLUSTERED kernel.  A cluster of CS CTAs works on super-tiles (class z, n-tile y, group of CS m-tiles):
// CTA r of the cluster owns m-tile CS*xs + r, and all CS CTAs need the SAME weight tiles in the same order.  Each
// k-block's weight tile (pre-split hi | lo, stored in global memory as the ready-made swizzled shared-memory image,
// tc_weights_kernel) is therefore fetched ONCE per cluster: CTA r bulk-copies slice r of it and the copy engine
// multicasts the slice into every CTA's stage, so a stage is free again only when the consumers of EVERY CTA of the
// cluster are done with it (each consumer warp arrives on the stage's empty barrier in all CTAs).
// The k-blocks of all super-tiles of a cluster form one stream through the stage ring; a chunk never spans two tiles.
template <int BN>
__global__ void __maxnreg__(168)     // 12 warps x 32 x 168 registers fit one SM
tc_tapgemm_kernel(const __grid_constant__ TapGemmParams p, const int mgroups, const int total_st) {
    using Cfg = TcCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int B_TILE_BYTES = Cfg::B_TILE_BYTES;
    constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;

    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES];     // A loader threads (cp.async completion) + weight bytes -> consumers
    __shared__ uint64_t empty_bar[STAGES];    // consumer warps of ALL CTAs of the cluster -> producers: stage is free everywhere

    const int tid = threadIdx.x;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform for the compiler
    const int ntn = p.N / BN;
    const int CS = (int)p.cluster;
    const int rank = CS > 1 ? (int)cluster_ctarank() : 0;
    const int cl_id = CS > 1 ? (int)cluster_id_x() : (int)blockIdx.x;
    const int cl_n = CS > 1 ? (int)cluster_count_x() : (int)gridDim.x;
    const uint16_t cl_mask = (uint16_t)((1u << CS) - 1u);
    // the dynamic shared window starts at the same offset in every CTA of the kernel, so the 1 KB-aligned base is
    // the same offset everywhere -- which the multicast copies rely on
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], kLoaderThreads + 1); mbar_init(&empty_bar[s], (uint32_t)(kConsumerWarps * CS)); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();             // peers' barriers are initialised before anything is sent to them

    // super-tile st -> (class z, m-group xs, n-tile y), n fastest: clusters running side by side share the A rows through L2
    auto st_z = [&](int st) { return st / (ntn * mgroups); };
    auto st_y = [&](int st) { return st % ntn; };
    auto st_m0 = [&](int st) { return (long long)(((st / ntn) % mgroups) * CS + rank) * TBM; };
    const int kb_per_tap = p.C / TBK;

    if (warp >= kLoaderWarp0) {
        // ================================ A loaders ================================
        // The tensor core reads only the TF32 bits of an fp32 operand (the 13 low mantissa bits are ignored; the parity
        // tests against float64 hold with the raw tensor as "hi"), so the raw fp32 activations ARE the "hi" operand; the "lo" operand (x - trunc(x)) comes from a
        // plane written by lo_plane_kernel before this launch.  A tile rows are therefore copied global -> swizzled
        // shared memory with cp.async (16 B per thread and row, zero-filled outside the image), completion is
        // counted on the stage's mbarrier (cp.async.mbarrier.arrive.noinc) -- no registers, no split, no stores,
        // no wait in the loader, which keeps the per-k-block instruction count of the loader warps small.
        const int tl = tid - kLoaderWarp0 * 32;      // 0..127
        const int a_chunk = tl & 7;
        // row r = tl/8 + 16*i lives at (r/8)*1024 + (r%8)*128 + ((chunk ^ r%8) * 16): i only moves the 1 KB group (2 per i)
        const uint32_t a_soff0 = (uint32_t)((tl >> 6) * 1024 + ((tl >> 3) & 7) * 128 + ((a_chunk ^ ((tl >> 3) & 7)) << 4));
        constexpr int RPT = TBM / (kLoaderThreads / 8);     // rows per thread: 8

        // ---- A cursor: 8 threads cover the 128 bytes of one row, 16 rows per pass, 8 passes
        int stA = cl_id, tapA = 0, cA = 0;
        int ntapsA = 0;
        int offA = 0;                           // taps[tapA].src_off + cA: float offset added to the row bases
        uint32_t tapbitA = 1u;
        const TapClass* clsA = &p.cls[0];
        uint32_t a_base[RPT];                     // float offset of the row's first tap position (< 2^31, checked at launch)
        uint32_t a_taps[RPT];                     // bit t: tap t of this row is inside the source image (0: row beyond M)
        auto setup_rows = [&]() {
            clsA = &p.cls[st_z(stA)];
            ntapsA = clsA->ntaps;
            const int Wo = clsA->Wo, HoWo = clsA->Ho * Wo;
            const long long M = (long long)p.batch * HoWo;
            const uint32_t wo_magic = (uint32_t)((0x100000000ull + (uint32_t)Wo - 1) / (uint32_t)Wo);   // exact for rem < 65536
            // first row by division, the others are 16 positions apart
            long long m = st_m0(stA) + (tl >> 3);
            int n = (int)(m / HoWo);
            int rem = (int)(m - (long long)n * HoWo);
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const bool ok = m < M;
                const int oy = (int)__umulhi((uint32_t)rem, wo_magic);
                const int ox = rem - oy * Wo;
                const int iy = oy * p.sstride, ix = ox * p.sstride;
                a_base[i] = (uint32_t)n * (uint32_t)p.src_img + (uint32_t)((iy * p.Ws + ix) * p.src_pitch + a_chunk * 4);
                uint32_t bits = 0xffffffffu;
                if (p.check) {
                    bits = 0u;
                    for (int t = 0; t < ntapsA; ++t)
                        if ((unsigned)(iy + clsA->taps[t].dy) < (unsigned)p.Hs && (unsigned)(ix + clsA->taps[t].dx) < (unsigned)p.Ws) bits |= 1u << t;
                }
                a_taps[i] = ok ? bits : 0u;
                m += 16; rem += 16;
                while (rem >= HoWo) { rem -= HoWo; ++n; }
            }
            offA = (int)clsA->taps[0].src_off;
            tapbitA = 1u;
        };
        if (stA < total_st) setup_rows();
        // copies the cursor's k-block into stage `stage` (hi = raw rows, lo = lo-plane rows) and advances the cursor
        auto issue_a = [&](uint32_t stage, uint64_t* full) {
            const uint32_t dst = stage + a_soff0;
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const bool v = (a_taps[i] & tapbitA) != 0u;
                const uint32_t off = v ? a_base[i] + (uint32_t)offA : 0u;
                const uint32_t bytes = (v && !(p.debug & 4)) ? 16u : 0u;   // 0: the 16 destination bytes are zero-filled
                if (p.debug & 2) continue;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + i * 2048), "l"(p.src + off), "r"(bytes) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + A_TILE_BYTES + i * 2048), "l"(p.src_lo + off), "r"(bytes) : "memory");
            }
            asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(full)) : "memory");
            cA += TBK; offA += TBK;
            if (cA == p.C) {
                cA = 0;
                if (++tapA == ntapsA) {
                    tapA = 0;
                    stA += cl_n;
                    if (stA < total_st) setup_rows();
                } else {
                    offA = (int)clsA->taps[tapA].src_off;
                    tapbitA <<= 1;
                }
            }
        };

        // weight tile of the cursor's k-block.  Global layout (tc_weights_kernel): per tap 2*N*C floats; inside, block
        // (n-tile y, k-block kc) holds the swizzled shared-memory image [hi: BN rows x 128 B | lo: BN rows x 128 B];
        // this CTA copies slice `rank` of it, multicast to every CTA of the cluster
        const uint32_t slice = (uint32_t)(2 * B_TILE_BYTES / CS);
        auto issue_b = [&](uint32_t stage, uint64_t* full) {
            if (p.debug & 8) { mbar_arrive(full); return; }      // timing decomposition: no weight copy
            mbar_expect_tx(full, (uint32_t)(2 * B_TILE_BYTES));
            const float* wt = p.wk_hi + 2 * clsA->taps[tapA].w_off + ((long long)st_y(stA) * kb_per_tap + cA / TBK) * (2 * BN * TBK);
            bulk_g2s(stage + 2 * A_TILE_BYTES + (uint32_t)rank * slice, reinterpret_cast<const char*>(wt) + (size_t)rank * slice,
                     slice, full, cl_mask, CS > 1);
        };

        // ---- copy stream: the loaders run ahead of the tensor core by as many k-blocks as there are free stages
        int sS = 0;                                 // stage of the next k-block and the parity its empty barrier
        uint32_t phS = 1;                           // shows once free (fresh barrier: parity 1 counts as complete)
        while (stA < total_st) {
            mbar_wait(&empty_bar[sS], phS);
            if (tl == 0) issue_b(smem_base + sS * STAGE_BYTES, &full_bar[sS]);
            issue_a(smem_base + sS * STAGE_BYTES, &full_bar[sS]);
            if (++sS == STAGES) { sS = 0; phS ^= 1u; }
        }
    } else {
        // ================================ wgmma consumers + epilogue ================================
        // warpgroup wg owns tile rows [64*wg, 64*wg + 64); thread layout of the accumulators: see wgmma_tf32
        constexpr int HALF = BN / 2;                 // accumulator registers per thread for a 64 x BN product
        const int wg = warp >> 2;
        float acc[HALF];                             // fp32 register accumulators of the tile (main + cross)
        float dm[HALF], dc[HALF];                    // chunk accumulators of the main and the cross terms
#pragma unroll
        for (int i = 0; i < HALF; ++i) { acc[i] = 0.f; dm[i] = 0.f; dc[i] = 0.f; }

        auto epilogue = [&](int st) {                // bias / ReLU / mask -> global, from the register accumulators
            const TapClass& cls = p.cls[st_z(st)];
            const int Wo = cls.Wo, HoWo = cls.Ho * Wo;
            const int col0 = st_y(st) * BN + 2 * (lane & 3);
            const int lcb = p.quad_lcb;              // log2(quad_cb)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const long long m = st_m0(st) + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
                if (m >= (long long)p.batch * HoWo) continue;
                const int n = (int)(m / HoWo);
                const int rem = (int)(m - (long long)n * HoWo);
                const int oy = rem / Wo;
                const int ox = rem - oy * Wo;
                // destination float offsets fit 32 bits (checked at launch)
                const uint32_t img = (uint32_t)n * (uint32_t)p.dst_img;
                const uint32_t off_plain = img + (uint32_t)(((oy * p.dstride + cls.py) * p.Wd + (ox * p.dstride + cls.px)) * p.dst_pitch);
                // groups of 4 column pairs, so that the ReLU-mask loads of a group are in flight together
                constexpr int NG = BN / 8;
                constexpr int GB = NG < 4 ? NG : 4;
#pragma unroll
                for (int j0 = 0; j0 < NG; j0 += GB) {
                    uint32_t offs[GB];
                    int chs[GB];
                    bool oks[GB];
                    float2 mks[GB];
#pragma unroll
                    for (int u = 0; u < GB; ++u) {
                        const int col = col0 + (j0 + u) * 8;
                        oks[u] = true;
                        if (p.quad) {
                            const int c = col >> lcb;
                            chs[u] = col & (p.quad_cb - 1);
                            const int y = oy * 2 + (c >> 1), x = ox * 2 + (c & 1);
                            oks[u] = y < p.Hd && x < p.Wd;
                            offs[u] = img + (uint32_t)((y * p.Wd + x) * p.dst_pitch + chs[u]);
                        } else {
                            chs[u] = col;
                            offs[u] = off_plain + (uint32_t)col;
                        }
                    }
                    if (p.mask) {
#pragma unroll
                        for (int u = 0; u < GB; ++u)
                            mks[u] = oks[u] ? __ldg(reinterpret_cast<const float2*>(p.mask + offs[u])) : make_float2(0.f, 0.f);
                    }
#pragma unroll
                    for (int u = 0; u < GB; ++u) {
                        if (!oks[u]) continue;
                        const int r = 4 * (j0 + u) + 2 * h;
                        float2 o = make_float2(acc[r], acc[r + 1]);
                        if (p.bias) {
                            const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + chs[u]));
                            o.x += b.x; o.y += b.y;
                        }
                        if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                        if (p.mask) { o.x = mks[u].x > 0.f ? o.x : 0.f; o.y = mks[u].y > 0.f ? o.y : 0.f; }
                        *reinterpret_cast<float2*>(p.dst + offs[u]) = o;
                        if (p.dst_lo != nullptr) {           // second TF32 operand of the consumer layer
                            float2 hi, lo;
                            split_tf32(o.x, hi.x, lo.x); split_tf32(o.y, hi.y, lo.y);
                            *reinterpret_cast<float2*>(p.dst_lo + offs[u]) = lo;
                        }
                    }
                }
            }
        };

        // stage s is free in this CTA's consumers: lane r < CS arrives on the stage's empty barrier of cluster CTA r
        auto release = [&](int s) {
            if (lane < CS) {
                if (CS > 1) mbar_arrive_cluster(&empty_bar[s], (uint32_t)lane);
                else mbar_arrive(&empty_bar[s]);
            }
        };

        int g = 0;                                   // k-blocks consumed so far (all tiles)
        for (int st = cl_id; st < total_st; st += cl_n) {
            const int nkb = p.cls[st_z(st)].ntaps * kb_per_tap;
            int prev = -1;                           // stage whose wgmma group may still be in flight
            for (int kb = 0; kb < nkb; ++kb, ++g) {
                const int s = g % STAGES;
                const uint32_t stage = smem_base + s * STAGE_BYTES;
                mbar_wait(&full_bar[s], (uint32_t)((g / STAGES) & 1));
                // the A rows were written by cp.async (generic proxy); wgmma reads through the async proxy
                fence_async_smem();
                const uint64_t a_hi = make_desc(stage + wg * (A_TILE_BYTES / 2));
                const uint64_t a_lo = make_desc(stage + A_TILE_BYTES + wg * (A_TILE_BYTES / 2));
                const uint64_t b_hi = make_desc(stage + 2 * A_TILE_BYTES);
                const uint64_t b_lo = make_desc(stage + 2 * A_TILE_BYTES + B_TILE_BYTES);
                // per 8-wide k-step:  main (+)= a_hi x b_hi,  cross (+)= a_hi x b_lo,  cross += a_lo x b_hi
                // (two disjoint accumulator arrays: wgmma groups writing overlapping register ranges are serialised)
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < TBK / 8; ++ks) {
                    const uint64_t adv = (uint64_t)(ks * 2);      // 32 bytes per k-step, in 16-byte units
                    const uint32_t keep = ((kb % CHUNK_KB) | ks) != 0 ? 1u : 0u;
                    wgmma_tf32<BN>(dm, a_hi + adv, b_hi + adv, keep);
                    wgmma_tf32<BN>(dc, a_hi + adv, b_lo + adv, keep);
                    wgmma_tf32<BN>(dc, a_lo + adv, b_hi + adv, 1u);
                }
                wgmma_commit();
                if (kb % CHUNK_KB == CHUNK_KB - 1 || kb == nkb - 1) {
                    wgmma_wait<0>();
                    fence_regs<HALF>(dm);
                    fence_regs<HALF>(dc);
                    if (prev >= 0) release(prev);
                    release(s);
                    prev = -1;
#pragma unroll
                    for (int i = 0; i < HALF; ++i) { acc[i] += dm[i]; acc[i] += dc[i]; }
                } else {
                    if (prev >= 0) { wgmma_wait<1>(); release(prev); }
                    prev = s;
                }
            }
            epilogue(st);
#pragma unroll
            for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
        }
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();             // nobody leaves while a peer may still multicast to / arrive on it
}

constexpr int tc_bn_slot(int BN) { return BN == 64 ? 1 : 0; }

template <int BN>
int32_t tc_launch_t(const TapGemmParams& p, int mgroups, int total_st, unsigned grid, cudaStream_t stream) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kTcThreads);
    cfg.dynamicSmemBytes = TcCfg<BN>::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)p.cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    CPB_CUDA(cudaLaunchKernelEx(&cfg, tc_tapgemm_kernel<BN>, p, mgroups, total_st));
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int BN>
int32_t tc_launch(const TapGemmParams& p0, cudaStream_t stream) {
    long long max_m = 0;
    for (int c = 0; c < p0.nclass; ++c) {
        long long m = (long long)p0.batch * p0.cls[c].Ho * p0.cls[c].Wo;
        if (m > max_m) max_m = m;
    }
    if (max_m == 0) return CPB_OK;
    TapGemmParams p = p0;
    p.cluster = g_tc_cluster;
    const long long mtiles = (max_m + TBM - 1) / TBM;
    const long long mgroups = (mtiles + p.cluster - 1) / p.cluster;
    const long long total_st = mgroups * (p.N / BN) * p.nclass;
    const int resident = g_tc_clusters[tc_bn_slot(BN)];
    CPB_REQUIRE(total_st < (1ll << 30) && resident > 0, "tc_tapgemm: bad tile count");
    CPB_REQUIRE((long long)p.batch * p.src_img < (1ll << 31) && (long long)p.batch * p.dst_img < (1ll << 31),
                "tc_tapgemm: tensors too large for 32-bit row offsets");
    for (int c = 0; c < p.nclass; ++c) CPB_REQUIRE(p.cls[c].ntaps <= 32, "tc_tapgemm: more than 32 taps");
    if (p.quad) {
        CPB_REQUIRE((p.quad_cb & (p.quad_cb - 1)) == 0, "tc_tapgemm: quad form needs a power-of-two channel count");
        p.quad_lcb = 0;
        while ((1 << p.quad_lcb) < p.quad_cb) ++p.quad_lcb;
    }
    const unsigned grid = (unsigned)((total_st < resident ? total_st : resident) * p.cluster);
    return tc_launch_t<BN>(p, (int)mgroups, (int)total_st, grid, stream);
}

template <int BN>
int32_t tc_init_one() {
    using Cfg = TcCfg<BN>;
    CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (g_tc_cluster > 1) CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    // how many clusters of this kernel are co-resident (GPC boundaries can strand SMs for cluster sizes > 1)
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(g_tc_cluster * 1024));
    cfg.blockDim = dim3(kTcThreads);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)g_tc_cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    int n = 0;
    CPB_CUDA(cudaOccupancyMaxActiveClusters(&n, tc_tapgemm_kernel<BN>, &cfg));
    CPB_REQUIRE(n > 0, "tc_tapgemm: no resident cluster of %d CTAs possible", g_tc_cluster);
    g_tc_clusters[tc_bn_slot(BN)] = n;
    return CPB_OK;
}

// lo[i] = x[i] - trunc_tf32(x[i]): the second TF32 operand of an activation tensor (the first is x itself)
__global__ void lo_plane_kernel(const float4* __restrict__ x, float4* __restrict__ lo, long long n4) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(x + i);
        float4 h, l;
        split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
        lo[i] = l;
    }
}

// weight preparation.  Logical operand: per tap a K-major [N][C] matrix.  Stored per tap as 2*N*C floats: for each
// (n-tile y of BN rows, k-block kc of 32 floats) one block [hi image | lo image], each image the BN x 128-byte
// SWIZZLE_128B shared-memory tile exactly as the tensor core reads it -- so a k-block's operand is ONE contiguous
// 2*BN*128-byte bulk copy (tc_tapgemm_kernel, weight-tile producer).
__global__ void tc_weights_kernel(const float* __restrict__ params, float* __restrict__ dst, const __grid_constant__ TcWeightTable t) {
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= t.total) return;
    int j = 0;
    while (j < t.njobs - 1 && idx >= t.jobs[j].count) { idx -= t.jobs[j].count; ++j; }
    const TcWeightJob& job = t.jobs[j];
    float x;
    int tap, n, c;          // logical coordinates of element idx
    if (job.mode == 0) {
        // plain K-major matrix [N][C], one tap
        tap = 0; n = (int)(idx / job.C); c = (int)(idx % job.C);
        x = params[job.src_off + idx];
    } else if (job.mode == 2) {
        // quad scatter form: logical [j][i][class*Cb + cb][cs]; class (py,px) uses kernel tap (py+2j, px+2i)
        const int w = (job.k + 1) / 2;
        const int cs = (int)(idx % job.cs);
        long long rest = idx / job.cs;
        const int ncol = (int)(rest % (4 * job.cb));
        rest /= (4 * job.cb);
        const int i = (int)(rest % w), jj = (int)(rest / w);
        const int cls = ncol / job.cb, cb = ncol - cls * job.cb;
        const int kh = (cls >> 1) + 2 * jj, kw = (cls & 1) + 2 * i;
        x = (kh < job.k && kw < job.k) ? params[job.src_off + (((long long)kh * job.k + kw) * job.cb + cb) * job.cs + cs] : 0.f;
        tap = jj * w + i; n = ncol; c = cs;
    } else {
        // gather form: logical [kh][cs][kw*Cb + cb]  <-  source [kh][kw][cb][cs]
        const int run = job.k * job.cb;
        const int cc = (int)(idx % run);
        const long long rest = idx / run;
        const int cs = (int)(rest % job.cs);
        const int kh = (int)(rest / job.cs);
        const int kw = cc / job.cb, cb = cc - kw * job.cb;
        x = params[job.src_off + (((long long)kh * job.k + kw) * job.cb + cb) * job.cs + cs];
        tap = kh; n = cs; c = cc;
    }
    const int BN = tc_bn(job.N);
    const int nn = n % BN, cc = c % TBK;
    const long long block = ((long long)tap * (job.N / BN) + n / BN) * (job.C / TBK) + c / TBK;
    const long long at = job.dst_hi + block * (2 * BN * TBK) + (nn >> 3) * 256 + (nn & 7) * 32 + ((((cc >> 2) ^ (nn & 7))) << 2) + (cc & 3);
    const float hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u);
    dst[at] = hi;
    dst[at + BN * TBK] = x - hi;
}

}  // namespace

int32_t tc_tapgemm_init() {
    const char* e = getenv("CPB_TC_CLUSTER");
    g_tc_cluster = e ? atoi(e) : 2;
    CPB_REQUIRE(g_tc_cluster == 1 || g_tc_cluster == 2 || g_tc_cluster == 4 || g_tc_cluster == 8, "CPB_TC_CLUSTER must be 1, 2, 4 or 8");
    CPB_TRY(tc_init_one<32>());
    CPB_TRY(tc_init_one<64>());
    return CPB_OK;
}

bool tc_tapgemm_supported(const TapGemmParams& p) {
    if (p.quad && (p.N != 4 * p.quad_cb || p.nclass != 1)) return false;
    return p.ybatch == 1 && p.C % TBK == 0 && (p.N == 32 || p.N % 64 == 0) && p.wk_hi != nullptr && p.wk_lo != nullptr && p.src_lo != nullptr;
}

int32_t launch_tc_tapgemm(const TapGemmParams& p, cudaStream_t stream) {
    CPB_REQUIRE(tc_tapgemm_supported(p), "tc_tapgemm: unsupported problem (C=%d, N=%d)", p.C, p.N);
    switch (tc_bn(p.N)) {
        case 64: return tc_launch<64>(p, stream);
        default: return tc_launch<32>(p, stream);
    }
}

int32_t launch_lo_plane(const float* x, float* lo, long long count, cudaStream_t stream) {
    CPB_REQUIRE(count % 4 == 0, "lo_plane: count must be a multiple of 4");
    if (count == 0) return CPB_OK;
    const long long n4 = count / 4;
    const long long want = (n4 + 255) / 256;
    lo_plane_kernel<<<(unsigned)(want < 132 * 16 ? want : 132 * 16), 256, 0, stream>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(lo), n4);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_tc_weights(const float* params, float* dst, const TcWeightTable& table, cudaStream_t stream) {
    if (table.total == 0) return CPB_OK;
    tc_weights_kernel<<<cdiv(table.total, 256), 256, 0, stream>>>(params, dst, table);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
