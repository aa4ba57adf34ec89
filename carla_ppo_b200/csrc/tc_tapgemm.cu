// Tensor-core tap-GEMM for sm_90a: the same contraction as tapgemm.cu, computed with wgmma.mma_async
// (kind tf32, fp32 accumulators in registers) using the error-compensated 3xTF32 split
//
//     a*b  ~=  a_hi*b_hi + a_lo*b_hi + a_hi*b_lo ,   x_hi = x with the 13 low mantissa bits cleared,  x_lo = x - x_hi
//
// so that results stay fp32-accurate (relative error ~1e-6; a single TF32 pass gives ~3e-4 and would break the
// 1e-5 parity bar).  Operands are staged in shared memory in the wgmma canonical K-major SWIZZLE_128B layout (rows of
// 32 floats = 128 B, 8-row groups of 1024 B, 16-byte chunk index XOR row%8):
//   * A (activations, gathered rows) : cp.async 16 B per thread and row of the raw fp32 tensor, zero-filled outside the
//                                      image, completion counted on the stage's mbarrier.  Each consumer thread reads
//                                      its register fragment of the k-block with ld.shared and splits it into hi / lo
//                                      itself; both feed wgmma from registers (RS form), so no lo plane of an
//                                      activation tensor ever exists in global memory;
//   * B (weights)                    : stored by tc_weights_kernel as ready-made swizzled tile images [hi | lo]; one
//                                      cp.async.bulk per k-block (multicast to the CTAs of a cluster).
// Persistent, warp-specialised kernel (see tc_tapgemm_kernel): two consumer warpgroups (64 tile rows each, 12 wgmma per
// 32-wide k-block in one commit group: main (+)= a_hi x b_hi, cross (+)= a_hi x b_lo, cross += a_lo x b_hi) and four
// A-loader warps, the first lane of which also issues the weight-tile copies.
//
// Accumulation.  The tensor core adds into its fp32 accumulator with truncation, which shrinks a long running sum
// systematically (relative bias growing linearly with K).  Two measures bring this back to fp32-FMA level:
//   * the cross terms (2^-11 of the main term) accumulate in their OWN registers, so they do not re-truncate the
//     large accumulator;
//   * wgmma accumulation only runs over chunks of 128 k (4 k-blocks); each finished chunk is added to per-thread fp32
//     register accumulators (round-to-nearest).
// The register accumulators feed the bias / ReLU / ReLU-mask epilogue directly.
//
// Single-pass variant (PASSES = 1, math mode 2): a*b ~= rna(a) * rna(b), both operands rounded to the nearest TF32
// value (the A fragment in registers, the weights by tc_weights_kernel), ONE wgmma per 8-wide k-step into the chunk
// accumulator, no cross terms; a stage holds A + the hi weight image only.  Relative error ~3e-4 per product, unbiased;
// the chunked accumulation into fp32 registers is the same as above.
#include "tapgemm.cuh"
#include "tc_common.cuh"

namespace cpb {

namespace {

using namespace tc;

template <int BN, int PASSES>
struct TcCfg {
    static constexpr int B_TILE_BYTES = BN * TBK * 4;
    static constexpr int B_IMAGES = PASSES == 3 ? 2 : 1;                    // weight images per k-block: [hi | lo] or [hi]
    static constexpr int STAGE_BYTES = A_TILE_BYTES + B_IMAGES * B_TILE_BYTES;   // raw A rows | weight image(s)
    static constexpr int STAGES = 200 * 1024 / STAGE_BYTES;                 // 3 passes: BN 64: 6, BN 32: 8; 1 pass: 8, 10
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;   // +1024: manual 1 KB alignment
};
constexpr int CHUNK_KB = 4;   // k-blocks accumulated by the tensor core before adding into the fp32 register accumulators

constexpr int kConsumerWarps = 8;                     // warps 0-7: two wgmma warpgroups + epilogue
constexpr int kLoaderWarp0 = 8;                       // warps 8-11: A loaders (cp.async)
constexpr int kLoaderWarps = 4;
constexpr int kLoaderThreads = kLoaderWarps * 32;
constexpr int kTcThreads = 384;                       // a multiple of 4 warps: registers are granted per 4 warps

int g_tc_cluster = 1;         // CTAs per cluster = multicast width of the weight tiles (CPB_TC_CLUSTER, 1/2/4/8)
int g_tc_clusters[2][2] = {{0, 0}, {0, 0}};   // co-resident clusters of the persistent grid, per instantiation [passes 3/1][BN 32/64]

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
// K-split (KSPLIT instantiations, p.ksplit > 1, dense problems): the work items are (super-tile, split) pairs, split
// fastest; item (st, ks) covers k-blocks [nkb*ks/ksplit, nkb*(ks+1)/ksplit) of the tile and stores its raw sums at
// p.dst + ks * p.kpartial_stride (the launcher points dst at the partial buffer and clears the epilogue).  Without
// KSPLIT the work items are the super-tiles and the split bookkeeping compiles away: the per-k-block loop of the
// unsplit kernels keeps its instructions and registers.
template <int BN, int PASSES, bool KSPLIT>
__global__ void __maxnreg__(168)     // 12 warps x 32 x 168 registers fit one SM
tc_tapgemm_kernel(const __grid_constant__ TapGemmParams p, const int mgroups, const int total_w) {
    static_assert(PASSES == 3 || PASSES == 1, "3xTF32 or a single TF32 pass");
    using Cfg = TcCfg<BN, PASSES>;
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
    const int ksplit = KSPLIT ? p.ksplit : 1;
    // first k-block of split ks of a tile with nkb k-blocks
    auto split_kb = [&](int nkb, int ks) { return (int)((long long)nkb * ks / ksplit); };

    if (warp >= kLoaderWarp0) {
        // ================================ A loaders ================================
        // The raw fp32 activation rows are copied global -> swizzled shared memory with cp.async (16 B per thread and
        // row, zero-filled outside the image); the consumers split them into TF32 hi / lo in registers.  Completion is
        // counted on the stage's mbarrier (cp.async.mbarrier.arrive.noinc) -- no registers, no stores, no wait in the
        // loader, which keeps the per-k-block instruction count of the loader warps small.
        const int tl = tid - kLoaderWarp0 * 32;      // 0..127
        const int a_chunk = tl & 7;
        // row r = tl/8 + 16*i lives at (r/8)*1024 + (r%8)*128 + ((chunk ^ r%8) * 16): i only moves the 1 KB group (2 per i)
        const uint32_t a_soff0 = (uint32_t)((tl >> 6) * 1024 + ((tl >> 3) & 7) * 128 + ((a_chunk ^ ((tl >> 3) & 7)) << 4));
        constexpr int RPT = TBM / (kLoaderThreads / 8);     // rows per thread: 8

        // ---- A cursor: 8 threads cover the 128 bytes of one row, 16 rows per pass, 8 passes
        int wA = cl_id, stA = 0, tapA = 0, cA = 0;   // work item, its super-tile, tap and k offset inside the tap
        int kbLeftA = 0;                        // k-blocks of the work item not yet issued
        int ntapsA = 0;
        int offA = 0;                           // taps[tapA].src_off + cA: float offset added to the row bases
        uint32_t tapbitA = 1u;
        const TapClass* clsA = &p.cls[0];
        uint32_t a_base[RPT];                     // float offset of the row's first tap position (< 2^31, checked at launch)
        uint32_t a_taps[RPT];                     // bit t: tap t of this row is inside the source image (0: row beyond M)
        auto setup_rows = [&]() {
            stA = KSPLIT ? wA / ksplit : wA;
            const int ksA = wA - stA * ksplit;
            clsA = &p.cls[st_z(stA)];
            ntapsA = clsA->ntaps;
            const int Wo = clsA->Wo, HoWo = clsA->Ho * Wo;
            const long long M = (long long)p.batch * HoWo;
            const uint32_t wo_magic = row_magic(Wo);
            // first row by division, the others are 16 positions apart
            long long m = st_m0(stA) + (tl >> 3);
            int n = (int)(m / HoWo);
            int rem = (int)(m - (long long)n * HoWo);
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const bool ok = m < M;
                const int oy = row_of(rem, wo_magic);
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
            if constexpr (KSPLIT) {
                const int nkb = ntapsA * kb_per_tap;
                const int kb0 = split_kb(nkb, ksA);
                kbLeftA = split_kb(nkb, ksA + 1) - kb0;
                tapA = kb0 / kb_per_tap;
                cA = (kb0 - tapA * kb_per_tap) * TBK;
                offA = (int)clsA->taps[tapA].src_off + cA;
                tapbitA = 1u << tapA;
            } else {
                offA = (int)clsA->taps[0].src_off;
                tapbitA = 1u;
            }
        };
        if (wA < total_w) setup_rows();
        // copies the cursor's k-block into stage `stage` and advances the cursor
        auto issue_a = [&](uint32_t stage, uint64_t* full) {
            const uint32_t dst = stage + a_soff0;
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const bool v = (a_taps[i] & tapbitA) != 0u;
                const uint32_t off = v ? a_base[i] + (uint32_t)offA : 0u;
                const uint32_t bytes = (v && !(p.debug & 4)) ? 16u : 0u;   // 0: the 16 destination bytes are zero-filled
                if (p.debug & 2) continue;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + i * 2048), "l"(p.src + off), "r"(bytes) : "memory");
            }
            asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(full)) : "memory");
            cA += TBK; offA += TBK;
            if constexpr (KSPLIT) {
                if (--kbLeftA == 0) {
                    wA += cl_n;
                    if (wA < total_w) setup_rows();
                } else if (cA == p.C) {
                    cA = 0;
                    ++tapA;
                    offA = (int)clsA->taps[tapA].src_off;
                    tapbitA <<= 1;
                }
            } else if (cA == p.C) {
                cA = 0;
                if (++tapA == ntapsA) {
                    tapA = 0;
                    wA += cl_n;
                    if (wA < total_w) setup_rows();
                } else {
                    offA = (int)clsA->taps[tapA].src_off;
                    tapbitA <<= 1;
                }
            }
        };

        // weight tile of the cursor's k-block.  Global layout (tc_weights_kernel): per tap 2*N*C floats; inside, block
        // (n-tile y, k-block kc) holds the swizzled shared-memory image [hi: BN rows x 128 B | lo: BN rows x 128 B]
        // (the single pass copies the hi image only); this CTA copies slice `rank` of it, multicast to every CTA of
        // the cluster
        constexpr int B_BYTES = Cfg::B_IMAGES * B_TILE_BYTES;
        const uint32_t slice = (uint32_t)(B_BYTES / CS);
        auto issue_b = [&](uint32_t stage, uint64_t* full) {
            if (p.debug & 8) { mbar_arrive(full); return; }      // timing decomposition: no weight copy
            mbar_expect_tx(full, (uint32_t)B_BYTES);
            const float* wt = p.wk_hi + 2 * clsA->taps[tapA].w_off + ((long long)st_y(stA) * kb_per_tap + cA / TBK) * (2 * BN * TBK);
            bulk_g2s(stage + A_TILE_BYTES + (uint32_t)rank * slice, reinterpret_cast<const char*>(wt) + (size_t)rank * slice,
                     slice, full, cl_mask, CS > 1);
        };

        // ---- copy stream: the loaders run ahead of the tensor core by as many k-blocks as there are free stages
        int sS = 0;                                 // stage of the next k-block and the parity its empty barrier
        uint32_t phS = 1;                           // shows once free (fresh barrier: parity 1 counts as complete)
        while (wA < total_w) {
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
        float dm[HALF], dc[HALF];                    // chunk accumulators of the main and the cross terms (3 passes)
#pragma unroll
        for (int i = 0; i < HALF; ++i) { acc[i] = 0.f; dm[i] = 0.f; dc[i] = 0.f; }

        auto epilogue = [&](int st, int ks) {        // bias / ReLU / mask -> global, from the register accumulators
            const TapClass& cls = p.cls[st_z(st)];
            float* const dst = KSPLIT ? p.dst + (long long)ks * p.kpartial_stride : p.dst;
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
                        *reinterpret_cast<float2*>(dst + offs[u]) = o;
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

        // A fragment of this thread (wgmma_tf32_rs): tile rows r0 = 64*wg + 16*(warp%4) + lane/4 and r0 + 8 (the next
        // 1 KB row group), k = lane%4 (+4) of each 8-wide k-step, i.e. 16-byte chunk 2*ks (+1) XOR r0%8 of the row.  The
        // 8 rows a warp reads at once sit in 8 different chunks, so the 32-bit shared loads are bank-conflict free.
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const uint32_t a_row = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + (lane & 3) * 4);
        const uint32_t a_swz = (uint32_t)((r0 & 7) << 4);

        int g = 0;                                   // k-blocks consumed so far (all tiles)
        for (int w = cl_id; w < total_w; w += cl_n) {
            const int st = KSPLIT ? w / ksplit : w, ks = KSPLIT ? w - st * ksplit : 0;
            const int nkb_tile = p.cls[st_z(st)].ntaps * kb_per_tap;
            const int nkb = KSPLIT ? split_kb(nkb_tile, ks + 1) - split_kb(nkb_tile, ks) : nkb_tile;
            for (int kb = 0; kb < nkb; ++kb, ++g) {
                const int s = g % STAGES;
                const uint32_t stage = smem_base + s * STAGE_BYTES;
                mbar_wait(&full_bar[s], (uint32_t)((g / STAGES) & 1));
                // the k-block's A fragment, split into TF32 hi / lo: ahi[ks][2*h + v], alo[ks][2*h + v]
                // (single pass: ahi = the fragment rounded to nearest TF32, no alo)
                uint32_t ahi[TBK / 8][4], alo[TBK / 8][4];
#pragma unroll
                for (int ks = 0; ks < TBK / 8; ++ks)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int v = 0; v < 2; ++v) {
                            float x;
                            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x)
                                         : "r"(stage + a_row + v * 1024 + ((uint32_t)((2 * ks + h) << 4) ^ a_swz)));
                            if constexpr (PASSES == 3) {
                                float hi, lo;
                                split_tf32(x, hi, lo);
                                ahi[ks][2 * h + v] = __float_as_uint(hi);
                                alo[ks][2 * h + v] = __float_as_uint(lo);
                            } else {
                                ahi[ks][2 * h + v] = round_tf32(x);
                            }
                        }
                // the split stays before the fence: ptxas serialises a wgmma stream in which a non-wgmma instruction
                // defines an A register while a group is in flight (C7513)
#pragma unroll
                for (int ks = 0; ks < TBK / 8; ++ks)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        if constexpr (PASSES == 3) asm volatile("" : "+r"(ahi[ks][i]), "+r"(alo[ks][i]));
                        else asm volatile("" : "+r"(ahi[ks][i]));
                    }
                const uint64_t b_hi = make_desc(stage + A_TILE_BYTES);
                const uint64_t b_lo = make_desc(stage + A_TILE_BYTES + B_TILE_BYTES);
                // per 8-wide k-step:  main (+)= a_hi x b_hi,  cross (+)= a_hi x b_lo,  cross += a_lo x b_hi, the whole
                // k-block as one commit group (single pass: main (+)= a x b only).  Two disjoint accumulator arrays: a
                // wgmma into a register range that only partly overlaps one in flight is serialised.  The group is
                // retired before the next k-block's split (see above); the other consumer warpgroup's group keeps the
                // tensor pipe busy meanwhile.
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < TBK / 8; ++ks) {
                    const uint64_t adv = (uint64_t)(ks * 2);      // 32 bytes per k-step, in 16-byte units
                    const uint32_t keep = ((kb % CHUNK_KB) | ks) != 0 ? 1u : 0u;
                    wgmma_tf32_rs<BN>(dm, ahi[ks], b_hi + adv, keep);
                    if constexpr (PASSES == 3) {
                        wgmma_tf32_rs<BN>(dc, ahi[ks], b_lo + adv, keep);
                        wgmma_tf32_rs<BN>(dc, alo[ks], b_hi + adv, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs<HALF>(dm);
                if constexpr (PASSES == 3) fence_regs<HALF>(dc);
                release(s);
                if (kb % CHUNK_KB == CHUNK_KB - 1 || kb == nkb - 1) {
#pragma unroll
                    for (int i = 0; i < HALF; ++i) {
                        acc[i] += dm[i];
                        if constexpr (PASSES == 3) acc[i] += dc[i];
                    }
                }
            }
            epilogue(st, ks);
#pragma unroll
            for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
        }
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();             // nobody leaves while a peer may still multicast to / arrive on it
}

constexpr int tc_bn_slot(int BN) { return BN == 64 ? 1 : 0; }
constexpr int tc_passes_slot(int PASSES) { return PASSES == 1 ? 1 : 0; }

template <int BN, int PASSES, bool KSPLIT>
int32_t tc_launch_t(const TapGemmParams& p, int mgroups, int total_w, unsigned grid, cudaStream_t stream) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kTcThreads);
    cfg.dynamicSmemBytes = TcCfg<BN, PASSES>::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)p.cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    CPB_CUDA(cudaLaunchKernelEx(&cfg, tc_tapgemm_kernel<BN, PASSES, KSPLIT>, p, mgroups, total_w));
    CPB_LAUNCHED();
    return CPB_OK;
}

template <int BN, int PASSES>
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
    const long long total_w = mgroups * (p.N / BN) * p.nclass * p.ksplit;
    const int resident = g_tc_clusters[tc_passes_slot(PASSES)][tc_bn_slot(BN)];
    CPB_REQUIRE(total_w < (1ll << 30) && resident > 0, "tc_tapgemm: bad tile count");
    CPB_REQUIRE(tc_offsets_fit(p.batch, p.src_img) && tc_offsets_fit(p.batch, p.dst_img),
                "tc_tapgemm: tensors too large for 32-bit row offsets");
    for (int c = 0; c < p.nclass; ++c) CPB_REQUIRE(p.cls[c].ntaps <= 32, "tc_tapgemm: more than 32 taps");
    if (p.quad) {
        CPB_REQUIRE((p.quad_cb & (p.quad_cb - 1)) == 0, "tc_tapgemm: quad form needs a power-of-two channel count");
        p.quad_lcb = 0;
        while ((1 << p.quad_lcb) < p.quad_cb) ++p.quad_lcb;
    }
    const unsigned grid = (unsigned)((total_w < resident ? total_w : resident) * p.cluster);
    if (p.ksplit == 1) return tc_launch_t<BN, PASSES, false>(p, (int)mgroups, (int)total_w, grid, stream);
    if constexpr (PASSES == 1) {
        // raw split sums into kpartial; the reduction adds them in split order and applies p's epilogue
        TapGemmParams q = p;
        q.dst = p.kpartial; q.bias = nullptr; q.mask = nullptr; q.relu = 0;
        CPB_TRY((tc_launch_t<BN, PASSES, true>(q, (int)mgroups, (int)total_w, grid, stream)));
        return launch_ksplit_reduce(p, stream);
    } else {
        CPB_REQUIRE(false, "tc_tapgemm: the k-split is built for the single TF32 pass only");
        return CPB_ERR_UNSUPPORTED;
    }
}

template <int BN, int PASSES>
int32_t tc_init_one() {
    using Cfg = TcCfg<BN, PASSES>;
    CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (g_tc_cluster > 1) CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    if constexpr (PASSES == 1) {   // the k-split variant: same threads and shared memory, so the same resident count
        CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        if (g_tc_cluster > 1) CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    }
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
    CPB_CUDA(cudaOccupancyMaxActiveClusters(&n, tc_tapgemm_kernel<BN, PASSES, false>, &cfg));
    CPB_REQUIRE(n > 0, "tc_tapgemm: no resident cluster of %d CTAs possible", g_tc_cluster);
    g_tc_clusters[tc_passes_slot(PASSES)][tc_bn_slot(BN)] = n;
    return CPB_OK;
}

// weight preparation.  Logical operand: per tap a K-major [N][C] matrix.  Stored per tap as 2*N*C floats: for each
// (n-tile y of BN rows, k-block kc of 32 floats) one block [hi image | lo image], each image the BN x 128-byte
// SWIZZLE_128B shared-memory tile exactly as the tensor core reads it -- so a k-block's operand is ONE contiguous
// 2*BN*128-byte bulk copy (tc_tapgemm_kernel, weight-tile producer).  job.round_nearest: hi = x rounded to the nearest
// TF32 value (the single-pass operand; the lo image is left unwritten) instead of x truncated.
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
    } else if (job.mode == 3) {
        // dense kernel stored [C][N]: strided reads (neighbouring n of later threads hit the same lines in L2),
        // coalesced image writes
        tap = 0; n = (int)(idx / job.C); c = (int)(idx % job.C);
        x = params[job.src_off + (long long)c * job.N + n];
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
    const float hi = job.round_nearest ? __uint_as_float(round_tf32(x)) : __uint_as_float(__float_as_uint(x) & 0xffffe000u);
    dst[at] = hi;
    if (!job.round_nearest) dst[at + BN * TBK] = x - hi;    // the single pass never reads the lo image
}

}  // namespace

int32_t tc_tapgemm_init() {
    const char* e = getenv("CPB_TC_CLUSTER");
    // default: no cluster.  Multicasting the weight tiles halves their L2 reads, but ties every stage of the CTAs of
    // a cluster to the slowest of their consumers, which costs more than the reads (measurements: DESIGN.md section 3)
    g_tc_cluster = e ? atoi(e) : 1;
    CPB_REQUIRE(g_tc_cluster == 1 || g_tc_cluster == 2 || g_tc_cluster == 4 || g_tc_cluster == 8, "CPB_TC_CLUSTER must be 1, 2, 4 or 8");
    CPB_TRY((tc_init_one<32, 3>()));
    CPB_TRY((tc_init_one<64, 3>()));
    CPB_TRY((tc_init_one<32, 1>()));
    CPB_TRY((tc_init_one<64, 1>()));
    return CPB_OK;
}

int tc_tapgemm_pick_ksplit(int K) {
    // splits of at most 320 k-blocks, at most 4 of them: the MlpVAE's 38 400-long reductions into 512 columns run as
    // 4 splits of 300 k-blocks, which at B = 512 (32 output tiles) fills the 132 SMs of an H100 SXM in one wave
    const int s = (int)cdiv(K / TBK, 320);
    return s < 1 ? 1 : (s > 4 ? 4 : s);
}

bool tc_tapgemm_supported(const TapGemmParams& p) {
    if (p.quad && (p.N != 4 * p.quad_cb || p.nclass != 1)) return false;
    if (p.ksplit < 1 || p.ksplit > kMaxKSplit) return false;
    // k-split: dense problems only (one output row per image), with room for the raw sums
    if (p.ksplit > 1 && (p.nclass != 1 || p.quad || p.cls[0].Ho != 1 || p.cls[0].Wo != 1 || p.dst_pitch != p.N ||
                         p.kpartial == nullptr || p.cls[0].ntaps * (p.C / TBK) < p.ksplit))
        return false;
    return p.ybatch == 1 && p.C % TBK == 0 && p.N % 32 == 0 && p.N > 0 && p.wk_hi != nullptr && p.wk_lo != nullptr;
}

int32_t launch_tc_tapgemm(const TapGemmParams& p, cudaStream_t stream) {
    CPB_REQUIRE(tc_tapgemm_supported(p), "tc_tapgemm: unsupported problem (C=%d, N=%d)", p.C, p.N);
    CPB_REQUIRE(p.passes == 3 || p.passes == 1, "tc_tapgemm: passes must be 3 or 1, got %d", p.passes);
    if (p.passes == 1) return tc_bn(p.N) == 64 ? tc_launch<64, 1>(p, stream) : tc_launch<32, 1>(p, stream);
    return tc_bn(p.N) == 64 ? tc_launch<64, 3>(p, stream) : tc_launch<32, 3>(p, stream);
}

int32_t launch_tc_weights(const float* params, float* dst, const TcWeightTable& table, cudaStream_t stream) {
    if (table.total == 0) return CPB_OK;
    tc_weights_kernel<<<cdiv(table.total, 256), 256, 0, stream>>>(params, dst, table);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
