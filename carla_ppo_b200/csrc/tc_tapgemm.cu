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
// 32-wide k-block in one commit group: main (+)= a_hi x b_hi, cross (+)= a_hi x b_lo, cross += a_lo x b_hi), four
// A-loader warps, the first lane of which also issues the weight-tile copies, and four epilogue warps: the consumers
// leave a finished tile's sums in a shared-memory buffer and start the next tile, the epilogue warps apply bias /
// ReLU / ReLU mask and store it with 16-byte accesses meanwhile.
//
// Accumulation.  The tensor core adds into its fp32 accumulator with truncation, which shrinks a long running sum
// systematically (relative bias growing linearly with K).  Two measures bring this back to fp32-FMA level:
//   * the cross terms (2^-11 of the main term) accumulate in their OWN registers, so they do not re-truncate the
//     large accumulator;
//   * wgmma accumulation only runs over chunks of 128 k (4 k-blocks); each finished chunk is added to per-thread fp32
//     accumulators (round-to-nearest): registers at BN 32 / 64; at BN 128, where they would not fit beside the chunk
//     accumulators, the thread's positions of the tile's output buffer in shared memory.
// These running sums are what the bias / ReLU / ReLU-mask epilogue receives.
//
// Single-pass variant (PASSES = 1, math mode 2): a*b ~= rna(a) * rna(b), both operands rounded to the nearest TF32
// value (the A fragment in registers, the weights by tc_weights_kernel), ONE wgmma per 8-wide k-step into the chunk
// accumulator, no cross terms; a stage holds A + the hi weight image only.  Relative error ~3e-4 per product, unbiased;
// the chunked accumulation into fp32 running sums is the same as above.
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
    static constexpr int OUT_BYTES = TBM * BN * 4;                          // the tile's raw sums, for the epilogue warps
    static constexpr int STAGES = (224 * 1024 - OUT_BYTES) / STAGE_BYTES;   // 3 passes: BN 128 / 64 / 32: 3 / 6 / 8; 1 pass: 5 / 8 / 10
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + OUT_BYTES + 1024;   // +1024: manual 1 KB alignment
    // registers per thread of each warpgroup role.  A 3-pass BN 128 consumer thread holds 128 chunk-accumulator and 32
    // A-fragment registers; below 192 ptxas serialises its wgmma (C7512).  Its loader and epilogue warpgroups fit in 56
    // and 72.  Every other instantiation: 168 / 80 / 80.  (The k-split variant runs at BN <= 64 only, see tc_bn.)
    static constexpr bool WIDE = BN == 128 && PASSES == 3;
    static constexpr int CONSUMER_REGS = WIDE ? 192 : 168, LOADER_REGS = WIDE ? 56 : 80, EPILOGUE_REGS = WIDE ? 72 : 80;
    static_assert(256 * CONSUMER_REGS + 128 * (LOADER_REGS + EPILOGUE_REGS) <= 512 * 128, "register file of one CTA");
};
constexpr int CHUNK_KB = 4;   // k-blocks accumulated by the tensor core before adding into the fp32 running sums

constexpr int kConsumerWarps = 8;                     // warps 0-7: two wgmma warpgroups
constexpr int kLoaderWarp0 = 8;                       // warps 8-11: A loaders (cp.async)
constexpr int kLoaderWarps = 4;
constexpr int kLoaderThreads = kLoaderWarps * 32;
constexpr int kEpilogueWarp0 = 12;                    // warps 12-15: tile epilogue (bias / ReLU / mask, global stores)
constexpr int kEpilogueWarps = 4;
constexpr int kEpilogueThreads = kEpilogueWarps * 32;
constexpr int kTcThreads = 512;                       // four warpgroups: setmaxnreg moves registers between whole warpgroups
// 512 threads start with kLaunchRegs registers each; setmaxnreg then shrinks the loader and the epilogue warpgroup and
// grows the two consumer warpgroups (TcCfg::*_REGS)
constexpr int kLaunchRegs = 128;
template <int R> __device__ __forceinline__ void reg_grow() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_shrink() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

int g_tc_cluster = 1;         // CTAs per cluster = multicast width of the weight tiles (CPB_TC_CLUSTER, 1/2/4/8)
int g_tc_clusters[2][3] = {};   // co-resident clusters of the persistent grid, per instantiation [passes 3/1][BN 32/64/128]

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
__global__ void __maxnreg__(kLaunchRegs)
tc_tapgemm_kernel(const __grid_constant__ TapGemmParams p, const int mgroups, const int total_w) {
    static_assert(PASSES == 3 || PASSES == 1, "3xTF32 or a single TF32 pass");
    using Cfg = TcCfg<BN, PASSES>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int B_TILE_BYTES = Cfg::B_TILE_BYTES;
    constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;

    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES];     // A loader threads (cp.async completion) + weight bytes -> consumers
    __shared__ uint64_t empty_bar[STAGES];    // consumer warps of ALL CTAs of the cluster -> producers: stage is free everywhere
    __shared__ uint64_t out_full;             // consumer warps -> epilogue warps: the tile's sums are in the output buffer
    __shared__ uint64_t out_empty;            // epilogue warps -> consumers: the output buffer has been read (CTA-local, both)

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
    // Output buffer (behind the stage ring): the tile's 128 x BN raw fp32 sums, rows of BN * 4 bytes, the 16-byte chunk
    // index of row r XORed with 2 * (r % 4).  A consumer warp's float2 fragment access covers rows g .. g+3 (per half
    // warp) x 32 bytes at the same columns, which the XOR spreads over all 32 banks; an epilogue thread's float4 read
    // stays inside one row, whose chunks the XOR only permutes.  Neither access has a bank conflict.  At BN 128 the
    // buffer is also where the consumers keep the running sums while the tile is accumulated.
    const uint32_t out_base = smem_base + STAGES * STAGE_BYTES;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], kLoaderThreads + 1); mbar_init(&empty_bar[s], (uint32_t)(kConsumerWarps * CS)); }
        mbar_init(&out_full, kConsumerWarps);
        mbar_init(&out_empty, kEpilogueWarps);
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

    if (warp >= kEpilogueWarp0) {
        reg_shrink<Cfg::EPILOGUE_REGS>();
        // ================================ tile epilogue ================================
        // The epilogue warps walk the same work items as the consumers.  Thread et owns 16-byte column chunk et % CPR of
        // tile rows et / CPR + RPP * i: a row's BN columns are contiguous in the destination (quad form: each parity
        // class's quad_cb >= 8 columns are), so a warp's stores and ReLU-mask loads are whole 128-byte lines.  The
        // destination offsets and the mask's sign bits of item w are computed / fetched while the consumers are still
        // accumulating w; once the sums arrive only shared loads, the arithmetic and the stores remain.
        constexpr int CPR = BN / 4;                        // 16-byte chunks per tile row
        constexpr int RPP = kEpilogueThreads / CPR;        // tile rows per pass of the four warps: 4 / 8 / 16 (BN 128 / 64 / 32)
        constexpr int NR = TBM / RPP;                      // rows per thread: 32 / 16 / 8
        constexpr uint32_t SKIP = 0xffffffffu;             // no destination: row beyond M or quad position outside the image
        const int et = tid - kEpilogueWarp0 * 32;
        const int ec = et % CPR, er = et / CPR;
        const uint32_t o_src = out_base + (uint32_t)(er * (BN * 4) + ((ec ^ ((er & 3) << 1)) << 4));   // RPP % 4 == 0: the XOR is the same for every i
        uint32_t phO = 0;                                  // parity of out_full's current phase
        for (int w = cl_id; w < total_w && !(p.debug & 16); w += cl_n) {
            const int st = KSPLIT ? w / ksplit : w, ks = KSPLIT ? w - st * ksplit : 0;
            const TapClass& cls = p.cls[st_z(st)];
            float* const dst = KSPLIT ? p.dst + (long long)ks * p.kpartial_stride : p.dst;
            const int Wo = cls.Wo, HoWo = cls.Ho * Wo;
            const uint32_t M = (uint32_t)p.batch * (uint32_t)HoWo;      // destination offsets fit 32 bits (checked at launch), so rows do
            const uint32_t wo_magic = row_magic(Wo);
            const int col = st_y(st) * BN + ec * 4;
            int ch = col, qy = 0, qx = 0;                  // quad form: column inside the parity class (qy, qx)
            if (p.quad) {
                const int c = col >> p.quad_lcb;
                ch = col & (p.quad_cb - 1);
                qy = c >> 1; qx = c & 1;
            }
            // row cursor: the first row by division, the others are RPP positions apart.  next_off returns the float
            // offset of the thread's chunk in the cursor's row (or SKIP) and moves the cursor on one pass
            const uint32_t m0 = (uint32_t)st_m0(st) + (uint32_t)er;
            const int n0 = (int)(m0 / (uint32_t)HoWo);
            const int rem0 = (int)(m0 - (uint32_t)n0 * (uint32_t)HoWo);
            uint32_t m = m0;
            int n = n0, rem = rem0;
            auto next_off = [&]() {
                const int oy = row_of(rem, wo_magic);
                const int ox = rem - oy * Wo;
                const uint32_t img = (uint32_t)n * (uint32_t)p.dst_img;
                bool ok = m < M;
                uint32_t off;
                if (p.quad) {
                    const int y = oy * 2 + qy, x = ox * 2 + qx;
                    ok = ok && y < p.Hd && x < p.Wd;
                    off = img + (uint32_t)((y * p.Wd + x) * p.dst_pitch + ch);
                } else {
                    off = img + (uint32_t)(((oy * p.dstride + cls.py) * p.Wd + (ox * p.dstride + cls.px)) * p.dst_pitch + col);
                }
                m += RPP; rem += RPP;
                while (rem >= HoWo) { rem -= HoWo; ++n; }
                return ok ? off : SKIP;
            };
            // ReLU mask: only the sign tests are kept, one word per eight rows, bit 4 * u + e = (mask element e of row u
            // of the eight) > 0.  keep[] is a queue: every trip pushes its words at the back, so that after the last
            // trip keep[0] belongs to the first eight rows (the loops stay rolled: a few hundred instructions, and a
            // bounded number of loads' registers at a time)
            uint32_t keep[NR / 8];
            if (p.mask) {
#pragma unroll 1
                for (int b = 0; b < NR / 8; ++b) {         // eight rows' loads in flight, one word per trip
                    uint32_t offs[8];
                    float4 mk[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) offs[u] = next_off();
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        mk[u] = offs[u] != SKIP ? __ldg(reinterpret_cast<const float4*>(p.mask + offs[u])) : make_float4(0.f, 0.f, 0.f, 0.f);
                    uint32_t bits = 0u;
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        bits |= ((mk[u].x > 0.f ? 1u : 0u) | (mk[u].y > 0.f ? 2u : 0u) | (mk[u].z > 0.f ? 4u : 0u) | (mk[u].w > 0.f ? 8u : 0u)) << (4 * u);
#pragma unroll
                    for (int q = 0; q < NR / 8 - 1; ++q) keep[q] = keep[q + 1];
                    keep[NR / 8 - 1] = bits;
                }
                m = m0; n = n0; rem = rem0;
            }
            float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.bias) bias = __ldg(reinterpret_cast<const float4*>(p.bias + ch));

            mbar_wait(&out_full, phO);
            phO ^= 1u;
#pragma unroll 1
            for (int b = 0; b < NR / 8; ++b) {
                uint32_t offs[8];
                float4 sums[8];
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(sums[u].x), "=f"(sums[u].y), "=f"(sums[u].z), "=f"(sums[u].w)
                                 : "r"(o_src + (uint32_t)((8 * b + u) * RPP * BN * 4)));
#pragma unroll
                for (int u = 0; u < 8; ++u) offs[u] = next_off();
                const uint32_t bits = p.mask ? keep[0] : 0u;
#pragma unroll
                for (int q = 0; q < NR / 8 - 1; ++q) keep[q] = keep[q + 1];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    if (offs[u] == SKIP) continue;
                    float4 o = sums[u];
                    if (p.bias) { o.x += bias.x; o.y += bias.y; o.z += bias.z; o.w += bias.w; }
                    if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                    if (p.mask) {
                        const uint32_t k = bits >> (4 * u);
                        o.x = (k & 1u) ? o.x : 0.f; o.y = (k & 2u) ? o.y : 0.f; o.z = (k & 4u) ? o.z : 0.f; o.w = (k & 8u) ? o.w : 0.f;
                    }
                    *reinterpret_cast<float4*>(dst + offs[u]) = o;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&out_empty);         // this warp has read its part of the buffer
        }
    } else if (warp >= kLoaderWarp0) {
        reg_shrink<Cfg::LOADER_REGS>();
        // ================================ A loaders ================================
        // The raw fp32 activation rows are copied global -> swizzled shared memory with cp.async (16 B per thread and
        // row, zero-filled outside the image); the consumers split them into TF32 hi / lo in registers.  Completion is
        // counted on the stage's mbarrier (cp.async.mbarrier.arrive.noinc) -- no registers, no stores, no wait in the
        // loader, which keeps the per-k-block instruction count of the loader warps small.
        const int tl = tid - kLoaderWarp0 * 32;      // 0..127
        const int a_chunk = tl & 7;
        // row r = tl/8 + 16*i lives at (r/8)*1024 + (r%8)*128 + ((chunk ^ r%8) * 16): i only moves the 1 KB group (2 per i)
        const uint32_t a_soff0 = (uint32_t)((tl >> 6) * 1024 + ((tl >> 3) & 7) * 128 + ((a_chunk ^ ((tl >> 3) & 7)) << 4));
        constexpr int RPP = kLoaderThreads / 8;             // rows per pass: 16
        constexpr int RPT = TBM / RPP;                      // rows per thread: 8

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
            // first row by division, the others are RPP positions apart
            long long m = st_m0(stA) + (tl >> 3);
            int n = (int)(m / HoWo);
            int rem = (int)(m - (long long)n * HoWo);
            int iy[RPT], ix[RPT];
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const int oy = row_of(rem, wo_magic);
                const int ox = rem - oy * Wo;
                iy[i] = oy * p.sstride; ix[i] = ox * p.sstride;
                a_base[i] = (uint32_t)n * (uint32_t)p.src_img + (uint32_t)((iy[i] * p.Ws + ix[i]) * p.src_pitch + a_chunk * 4);
                a_taps[i] = m < M ? 0xffffffffu : 0u;
                m += RPP; rem += RPP;
                while (rem >= HoWo) { rem -= HoWo; ++n; }
            }
            if (p.check) {
                // taps outside, rows inside: a tap's displacement is read once for the thread's RPT rows
                uint32_t in[RPT];
#pragma unroll
                for (int i = 0; i < RPT; ++i) in[i] = 0u;
                for (int t = 0; t < ntapsA; ++t) {
                    const int dy = clsA->taps[t].dy, dx = clsA->taps[t].dx;
#pragma unroll
                    for (int i = 0; i < RPT; ++i)
                        if ((unsigned)(iy[i] + dy) < (unsigned)p.Hs && (unsigned)(ix[i] + dx) < (unsigned)p.Ws) in[i] |= 1u << t;
                }
#pragma unroll
                for (int i = 0; i < RPT; ++i) a_taps[i] &= in[i];
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
        // ================================ wgmma consumers ================================
        reg_grow<Cfg::CONSUMER_REGS>();
        // warpgroup wg owns tile rows [64*wg, 64*wg + 64); thread layout of the accumulators: see wgmma_tf32
        constexpr int HALF = BN / 2;                 // accumulator registers per thread for a 64 x BN product
        constexpr bool SACC = BN == 128;             // the running sums live in the output buffer, not in registers
        const int wg = warp >> 2;
        float acc[SACC ? 1 : HALF];                  // BN 32 / 64: fp32 register running sums of the tile (main + cross)
        float dm[HALF], dc[HALF];                    // chunk accumulators of the main and the cross terms (3 passes)
#pragma unroll
        for (int i = 0; i < HALF; ++i) { dm[i] = 0.f; dc[i] = 0.f; }
        if constexpr (!SACC) {
#pragma unroll
            for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
        }

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
        // a_row addresses chunk 0 XOR r0%8; a stage is 1 KB aligned, so chunk c is (stage + a_row) ^ (c << 4).
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const uint32_t a_row = (uint32_t)((r0 >> 3) * 1024 + (r0 & 7) * 128 + ((r0 & 7) << 4) + (lane & 3) * 4);

        // The finished tile goes to the epilogue warps through the output buffer: acc[4*j + 2*h + c] is row r0 + 8*h,
        // columns 8*j + 2*(lane%4) + c, i.e. bytes 8*(lane%4) of the 32-byte pair of chunks j XOR r0%4 (layout: see
        // out_base).  The consumers then go straight on to the next item's first k-block.  At BN 128 the sums are
        // already there (same positions) and only the arrival on out_full remains.
        const uint32_t o_dst = (uint32_t)(r0 * (BN * 4) + ((r0 & 3) << 5) + (lane & 3) * 8);
        uint32_t phE = 1;                            // parity out_empty shows once free (fresh barrier: 1 counts as complete)
        auto hand_off = [&]() {
            mbar_wait(&out_empty, phE);
            phE ^= 1u;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(out_base + (uint32_t)(h * 8 * BN * 4) + (o_dst ^ (uint32_t)(j << 5))),
                                 "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1]) : "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&out_full);
        };

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
                uint32_t a_at = stage + a_row;       // opaque: one XOR per load rather than 8 chunk offsets held in registers
                asm volatile("" : "+r"(a_at));
#pragma unroll
                for (int ks = 0; ks < TBK / 8; ++ks)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int v = 0; v < 2; ++v) {
                            float x;
                            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x)
                                         : "r"((a_at ^ (uint32_t)((2 * ks + h) << 4)) + (uint32_t)(v * 1024)));
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
                    if constexpr (SACC) {
                        // read-modify-write of the thread's running sums in the output buffer, eight float2 loads in
                        // flight at a time.  The item's first chunk writes 0 + chunk (the register sums' first add,
                        // signed zeros included) once the epilogue warps have read the previous item's sums: a whole
                        // chunk after the previous item's out_full, which gives them that long to drain the buffer.
                        const bool first = kb < CHUNK_KB;
                        if (first && !(p.debug & 16)) {
                            mbar_wait(&out_empty, phE);
                            phE ^= 1u;
                        }
                        // out_base is 1 KB aligned, so pair j of the thread's row is (out_base + o_dst) ^ (j << 5): one
                        // XOR per access on a base made opaque here, instead of 16 pair addresses held in registers
                        // across the k-loop
                        uint32_t ob = out_base + o_dst;
                        asm volatile("" : "+r"(ob));
#pragma unroll
                        for (int j0 = 0; j0 < BN / 8; j0 += 4) {
                            float sum[4][2][2];
#pragma unroll
                            for (int j = 0; j < 4; ++j)
#pragma unroll
                                for (int h = 0; h < 2; ++h) {
                                    sum[j][h][0] = 0.f; sum[j][h][1] = 0.f;
                                    if (!first)
                                        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(sum[j][h][0]), "=f"(sum[j][h][1])
                                                     : "r"((ob ^ (uint32_t)((j0 + j) << 5)) + (uint32_t)(h * 8 * BN * 4)) : "memory");
                                }
#pragma unroll
                            for (int j = 0; j < 4; ++j)
#pragma unroll
                                for (int h = 0; h < 2; ++h) {
#pragma unroll
                                    for (int c = 0; c < 2; ++c) {
                                        sum[j][h][c] += dm[4 * (j0 + j) + 2 * h + c];
                                        if constexpr (PASSES == 3) sum[j][h][c] += dc[4 * (j0 + j) + 2 * h + c];
                                    }
                                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};"
                                                 ::"r"((ob ^ (uint32_t)((j0 + j) << 5)) + (uint32_t)(h * 8 * BN * 4)),
                                                 "f"(sum[j][h][0]), "f"(sum[j][h][1]) : "memory");
                                }
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < HALF; ++i) {
                            acc[i] += dm[i];
                            if constexpr (PASSES == 3) acc[i] += dc[i];
                        }
                    }
                }
            }
            if constexpr (SACC) {
                if (!(p.debug & 16)) {               // timing decomposition: no epilogue
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&out_full);
                }
            } else {
                if (!(p.debug & 16)) hand_off();     // timing decomposition: no epilogue
#pragma unroll
                for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
            }
        }
    }
    __syncthreads();
    if (CS > 1) cluster_sync_all();             // nobody leaves while a peer may still multicast to / arrive on it
}

constexpr int tc_bn_slot(int BN) { return BN == 128 ? 2 : (BN == 64 ? 1 : 0); }
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
    // the epilogue warps store (and read the bias and the ReLU mask) 16 bytes at a time
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
    CPB_REQUIRE(al16(p.dst) && al16(p.mask) && al16(p.bias) && p.dst_pitch % 4 == 0 && p.dst_img % 4 == 0 &&
                    (p.ksplit == 1 || (al16(p.kpartial) && p.kpartial_stride % 4 == 0)),
                "tc_tapgemm: destination, mask and bias must be 16-byte aligned");
    for (int c = 0; c < p.nclass; ++c) CPB_REQUIRE(p.cls[c].ntaps <= 32, "tc_tapgemm: more than 32 taps");
    if (p.quad) {
        CPB_REQUIRE((p.quad_cb & (p.quad_cb - 1)) == 0, "tc_tapgemm: quad form needs a power-of-two channel count");
        p.quad_lcb = 0;
        while ((1 << p.quad_lcb) < p.quad_cb) ++p.quad_lcb;
    }
    const unsigned grid = (unsigned)((total_w < resident ? total_w : resident) * p.cluster);
    if (p.ksplit == 1) return tc_launch_t<BN, PASSES, false>(p, (int)mgroups, (int)total_w, grid, stream);
    if constexpr (PASSES == 1 && BN <= 64) {
        // raw split sums into kpartial; the reduction adds them in split order and applies p's epilogue
        TapGemmParams q = p;
        q.dst = p.kpartial; q.bias = nullptr; q.mask = nullptr; q.relu = 0;
        CPB_TRY((tc_launch_t<BN, PASSES, true>(q, (int)mgroups, (int)total_w, grid, stream)));
        return launch_ksplit_reduce(p, stream);
    } else {
        CPB_REQUIRE(false, "tc_tapgemm: the k-split is built for the single TF32 pass at BN <= 64 only");
        return CPB_ERR_UNSUPPORTED;
    }
}

template <int BN, int PASSES>
int32_t tc_init_one() {
    using Cfg = TcCfg<BN, PASSES>;
    CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    if (g_tc_cluster > 1) CPB_CUDA(cudaFuncSetAttribute(tc_tapgemm_kernel<BN, PASSES, false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    if constexpr (PASSES == 1 && BN <= 64) {   // the k-split variant: same threads and shared memory, so the same resident count
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
    const int BN = tc_bn(job.N, job.ksplit != 0);
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
    CPB_TRY((tc_init_one<128, 3>()));
    CPB_TRY((tc_init_one<32, 1>()));
    CPB_TRY((tc_init_one<64, 1>()));
    CPB_TRY((tc_init_one<128, 1>()));
    return CPB_OK;
}

int tc_tapgemm_pick_ksplit(int K) {
    // splits of at most 320 k-blocks, at most 4 of them: the MlpVAE's 38 400-long reductions into 512 columns run as
    // 4 splits of 300 k-blocks, which at B = 512 (32 output tiles of 128 x 64: k-split problems stay at BN 64, see
    // tc_bn) fills the 132 SMs of an H100 SXM in one wave
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
    const int bn = tc_bn(p.N, p.ksplit > 1);
    if (p.passes == 1) return bn == 128 ? tc_launch<128, 1>(p, stream) : bn == 64 ? tc_launch<64, 1>(p, stream) : tc_launch<32, 1>(p, stream);
    return bn == 128 ? tc_launch<128, 3>(p, stream) : bn == 64 ? tc_launch<64, 3>(p, stream) : tc_launch<32, 3>(p, stream);
}

int32_t launch_tc_weights(const float* params, float* dst, const TcWeightTable& table, cudaStream_t stream) {
    if (table.total == 0) return CPB_OK;
    tc_weights_kernel<<<cdiv(table.total, 256), 256, 0, stream>>>(params, dst, table);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb
