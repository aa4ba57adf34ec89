// Tensor-core weight gradient for sm_90a (tf Conv2DBackpropFilter for conv and transposed-conv layers):
//
//   gw[i, j] = sum_{m}  big[row(m) + tap_off[i / run] + i % run] * small[m * J + j]        (same contract as wgrad.cu)
//
// as D[128 x BN] += A^T B with the REDUCTION index m on the MMA K axis.  In NHWC memory the channel index -- not m --
// is contiguous, while wgmma takes shared-memory TF32 operands only K-major.
// A (big, 128 channels i) goes to the tensor core from registers (RS-form wgmma), so it needs no K-major tile: warps
// 8-11 copy the raw fp32 rows "32 channels x 4 B at one reduction position" with cp.async (16 B per thread, zero-
// filled beyond len or I; completion counted on the stage's full barrier), eight consecutive positions per thread, so
// the position cursor advances by one position without divisions.  The A tile of a stage is position-major: row p
// (512 B) holds the 128 channels at position p, 16-byte chunk c XOR 4*(p % 2).  The MMA thread reads its fragment --
// tile rows g and g+8 of its warp's 16 (g = lane/4), k-columns t and t+4 of each 8-wide k-step (t = lane%4) -- as one
// ld.shared.v2 per reduction position: tile row 16*w + g + 8*v holds channel 16*w + 2*g + v, so the two rows are
// adjacent channels, and the chunk swizzle puts the two position parities of a warp load in different bank halves
// (two wavefronts, conflict-free).  It splits the fragment into TF32 hi / lo right before the k-block's wgmma.
// B (small, BN channels j) is staged by the same warps: 4 x LDG.128 of 4 channels at 4 consecutive reduction positions,
// a 4x4 register transpose into "one channel x 4 positions", the split and ONE 16-byte chunk per channel and part
// into the K-major SWIZZLE_128B tile (8 STS.128); tile row (BN/4)*c + cg holds channel 4*cg + c, so that a
// quarter-warp's stores are conflict-free.  Four B k-blocks are in flight per loader thread.
// Warps 0-7 (two warpgroups of 64 tile rows) issue the wgmma and store the partial, un-permuting rows and columns.
// 3xTF32 products, the separate cross-term registers, the chunked accumulation into fp32 register accumulators and the
// retirement of the RS group before the next fragment is split are those of tc_tapgemm.cu.  Each (i-tile, j-tile,
// split) CTA of the single split-K wave writes its partial [128 x BN] block; reduce_partials() sums the splits in a
// fixed order (deterministic).
// Single-pass variant (PASSES = 1, math mode 2): both operands are rounded to the nearest TF32 value, B stores the hi
// tile only, one wgmma per 8-wide k-step into the chunk accumulator, no cross terms.
#include "tc_common.cuh"
#include "wgrad.cuh"

namespace cpb {

namespace {

using namespace tc;

constexpr int CHUNK_KB = 4;

template <int BN, int PASSES>
struct TcWgCfg {
    static constexpr int B_TILE_BYTES = BN * TBK * 4;
    static constexpr int PARTS = PASSES == 3 ? 2 : 1;                // B tiles per stage: [hi | lo] or [hi]
    static constexpr int B_OFF = A_TILE_BYTES;                       // stage layout: raw A tile | B tile(s)
    static constexpr int STAGE_BYTES = A_TILE_BYTES + PARTS * B_TILE_BYTES;
    static constexpr int STAGES = (192 * 1024) / STAGE_BYTES < 8 ? (192 * 1024) / STAGE_BYTES : 8;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
};

constexpr int kWgMmaWarps = 8;                            // warps 0-7: wgmma, partial store
constexpr int kWgLoaderWarps = 4;                         // warps 8-11: A copies, B loads / stores
constexpr int kWgLoaderThreads = kWgLoaderWarps * 32;
constexpr int kWgThreads = (kWgMmaWarps + kWgLoaderWarps) * 32;

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
    __shared__ uint64_t full_bar[STAGES];     // loader threads' A copies (cp.async completion) + B warps -> wgmma
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
    // k-blocks of this split, rounded up to an even count (the chunk boundaries and the zero padding k-block of the
    // earlier two-k-blocks-per-iteration loop are kept, so the sums are unchanged bit for bit)
    const int nkb = m_end > m_begin ? 2 * (int)((m_end - m_begin + 2 * TBK - 1) / (2 * TBK)) : 0;

    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], kWgLoaderThreads + kWgLoaderWarps); mbar_init(&empty_bar[s], kWgMmaWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int len = (int)(m_end - m_begin);          // reduction positions of this split

    if (warp >= kWgMmaWarps) {
        // ================================ loaders ================================
        const int tl = tid - kWgMmaWarps * 32;       // 0..127
        // ---- A: thread = (16-byte chunk `lane` of the 128 channels, positions 8*pg .. 8*pg + 7 of each k-block)
        const int pg = tl >> 5;
        const int a_i = i0 + 4 * lane;
        const bool a_col_ok = a_i < p.I;
        long long a_coloff = 0;
        if (a_col_ok) {
            const int tap = a_i / p.run;
            a_coloff = p.tap_off[tap] + (a_i - tap * p.run);
        }
        const uint32_t a_dst0 = (uint32_t)(8 * pg * 512);
        // position cursor of this thread's NEXT copy: image n, position rem = oy*Wo + ox inside it.  Advancing by a
        // k-block (32 positions) needs no division: oy comes from a multiply-high (row_of).
        const uint32_t wo_magic = row_magic(p.Wo);
        const int dx = p.sstride * p.big_pitch;                              // next position in the row
        const int drow = (p.sstride * p.Wb - p.Wo * p.sstride) * p.big_pitch;   // ... wrapping to the next row
        const int dimg = (int)(p.big_img - (long long)p.Ho * p.sstride * p.Wb * p.big_pitch);   // ... to the next image
        int nA, remA, relA = 8 * pg;                               // relA: position index relative to m_begin
        {
            const long long m = m_begin + relA;
            nA = (int)(m / HoWo);
            remA = (int)(m - (long long)nA * HoWo);
        }
        auto issue_a = [&](uint32_t stage, uint64_t* full) {
            int oy = row_of(remA, wo_magic);
            int ox = remA - oy * p.Wo;
            uint32_t off = (uint32_t)nA * (uint32_t)p.big_img + (uint32_t)((oy * p.sstride * p.Wb + ox * p.sstride) * p.big_pitch) + (uint32_t)a_coloff;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const bool v = relA + j < len && a_col_ok;
                const uint32_t dst = stage + a_dst0 + j * 512 + ((lane ^ ((j & 1) << 2)) << 4);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(p.big + (v ? off : 0u)), "r"(v ? 16u : 0u) : "memory");
                off += (uint32_t)dx;
                if (++ox == p.Wo) { ox = 0; off += (uint32_t)drow; if (++oy == p.Ho) { oy = 0; off += (uint32_t)dimg; } }
            }
            asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(full)) : "memory");
            relA += TBK;
            remA += TBK;
            while (remA >= HoWo) { remA -= HoWo; ++nA; }
        };

        // ---- B: thread = (channel group of 4 output channels) x (position block of 4 reduction positions), a
        // quarter-warp covering 8 consecutive channel groups of ONE position (a contiguous 128-byte line per
        // LDG.128); BN = 32 leaves half of the threads idle.
        constexpr int BQ = BN / 4;                   // channel groups of the B tile
        constexpr int NCGH = BQ >= 8 ? BQ / 8 : 1;
        const int r = tl >> 3;                                     // 0..15
        const int cgb = (r % NCGH) * 8 + (lane & 7);
        const int mb0 = r / NCGH;                                  // BN 32: 0..15 (>= 8 idle), 64: 0..7
        const bool active = mb0 < 8;
        uint32_t soffb[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int rb = BQ * c + cgb;
            soffb[c] = (uint32_t)((rb >> 3) * 1024 + (rb & 7) * 128 + ((mb0 ^ (rb & 7)) << 4));
        }
        // 4x4 register transpose + split + store: x[j] = 4 channels at position j  ->  one chunk per channel
        // (single pass: rounded to nearest TF32, hi tile only)
        auto store_t = [&](uint32_t tile_hi, uint32_t tile_lo, const float4* x) {
            const float xs[4][4] = {{x[0].x, x[1].x, x[2].x, x[3].x}, {x[0].y, x[1].y, x[2].y, x[3].y},
                                    {x[0].z, x[1].z, x[2].z, x[3].z}, {x[0].w, x[1].w, x[2].w, x[3].w}};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if constexpr (PASSES == 3) {
                    float4 hi, lo;
                    split_tf32(xs[c][0], hi.x, lo.x); split_tf32(xs[c][1], hi.y, lo.y);
                    split_tf32(xs[c][2], hi.z, lo.z); split_tf32(xs[c][3], hi.w, lo.w);
                    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(tile_hi + soffb[c]), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
                    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(tile_lo + soffb[c]), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
                } else {
                    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(tile_hi + soffb[c]), "r"(round_tf32(xs[c][0])),
                                 "r"(round_tf32(xs[c][1])), "r"(round_tf32(xs[c][2])), "r"(round_tf32(xs[c][3])) : "memory");
                }
            }
        };
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
        float4 xb0[4], xb1[4], xb2[4], xb3[4];
        int sS = 0;
        uint32_t phS = 1;
        auto step = [&](int kb, float4* xb) {
            if (kb >= nkb) return;
            const uint32_t stage = smem_base + sS * STAGE_BYTES;
            mbar_wait(&empty_bar[sS], phS);
            issue_a(stage, &full_bar[sS]);
            if (active) store_t(stage + B_OFF, stage + B_OFF + B_TILE_BYTES, xb);
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[sS]);
            if (kb + 4 < nkb) load_b(xb);
            if (++sS == STAGES) { sS = 0; phS ^= 1u; }
        };
        if (nkb > 0) load_b(xb0);
        if (nkb > 1) load_b(xb1);
        if (nkb > 2) load_b(xb2);
        if (nkb > 3) load_b(xb3);
        for (int kb = 0; kb < nkb; kb += 4) {
            step(kb, xb0);
            step(kb + 1, xb1);
            step(kb + 2, xb2);
            step(kb + 3, xb3);
        }
    } else {
        // ================================ wgmma / partial store ================================
        // A fragment of this thread (wgmma_tf32_rs): tile rows 16*warp + g + 8*v (v = 0, 1) = channels
        // i0 + 16*warp + 2*g + v, k-columns t + 4*h + 8*ks = reduction positions p = t + 4*h + 8*ks of the k-block:
        // the float2 at row p, chunk (4*warp + g/2) XOR 4*(t % 2), byte 8*(g % 2)
        const int g = lane >> 2, t = lane & 3;
        const uint32_t a_rd = (uint32_t)(t * 512 + (((4 * warp + (g >> 1)) ^ ((t & 1) << 2)) << 4) + (g & 1) * 8);
        constexpr int HALF = BN / 2;                 // accumulator registers per thread for a 64 x BN product
        constexpr int DN = PASSES == 3 ? BN : HALF;
        float acc[HALF];                             // fp32 register accumulators (main + cross)
        float d[DN];                                 // chunk accumulators: [main (HALF) | cross (HALF, 3 passes only)]
#pragma unroll
        for (int i = 0; i < HALF; ++i) acc[i] = 0.f;
#pragma unroll
        for (int i = 0; i < DN; ++i) d[i] = 0.f;

        int s = 0;
        uint32_t ph = 0;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&full_bar[s], ph);
            const uint32_t stage = smem_base + s * STAGE_BYTES;
            // the k-block's A fragment, split into TF32 hi / lo: ah[ks][2*h + v], al[ks][2*h + v]
            // (single pass: ah = the fragment rounded to nearest TF32, no al)
            uint32_t ah[TBK / 8][4], al[TBK / 8][4];
#pragma unroll
            for (int ks = 0; ks < TBK / 8; ++ks)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float2 x;
                    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(x.x), "=f"(x.y) : "r"(stage + a_rd + (4 * h + 8 * ks) * 512));
#pragma unroll
                    for (int v = 0; v < 2; ++v) {
                        const float xv = v ? x.y : x.x;
                        if constexpr (PASSES == 3) {
                            float hi, lo;
                            split_tf32(xv, hi, lo);
                            ah[ks][2 * h + v] = __float_as_uint(hi);
                            al[ks][2 * h + v] = __float_as_uint(lo);
                        } else {
                            ah[ks][2 * h + v] = round_tf32(xv);
                        }
                    }
                }
            // the split stays before the fence: ptxas serialises a wgmma stream in which a non-wgmma instruction
            // defines an A register while a group is in flight (C7513)
#pragma unroll
            for (int ks = 0; ks < TBK / 8; ++ks)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if constexpr (PASSES == 3) asm volatile("" : "+r"(ah[ks][i]), "+r"(al[ks][i]));
                    else asm volatile("" : "+r"(ah[ks][i]));
                }
            const uint64_t b_hi = make_desc(stage + B_OFF);
            const uint64_t b_lo = make_desc(stage + B_OFF + B_TILE_BYTES);
            // main (+)= a_hi x b_hi,  cross (+)= a_hi x b_lo,  cross += a_lo x b_hi (single pass: main (+)= a x b only),
            // the whole k-block as one commit group, retired before the next k-block's split; the other warpgroup's
            // group keeps the tensor pipe busy meanwhile.  Each product writes exactly one of the two disjoint
            // accumulator arrays: a wgmma into a register range that only partly overlaps one in flight is serialised.
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < TBK / 8; ++ks) {
                const uint64_t adv = (uint64_t)(ks * 2);          // 32 bytes per k-step (K-major)
                const uint32_t keep = ((kb % CHUNK_KB) | ks) != 0 ? 1u : 0u;
                wgmma_tf32_rs<BN>(d, ah[ks], b_hi + adv, keep);
                if constexpr (PASSES == 3) {
                    wgmma_tf32_rs<BN>(d + HALF, ah[ks], b_lo + adv, keep);
                    wgmma_tf32_rs<BN>(d + HALF, al[ks], b_hi + adv, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<DN>(d);
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            if (kb % CHUNK_KB == CHUNK_KB - 1 || kb == nkb - 1) {
#pragma unroll
                for (int i = 0; i < HALF; ++i) {
                    acc[i] += d[i];
                    if constexpr (PASSES == 3) acc[i] += d[HALF + i];
                }
            }
            if (++s == STAGES) { s = 0; ph ^= 1u; }
        }

        // ---- partial[split][i][j]: tile row 16*warp + g + 8*h holds channel i = i0 + 16*warp + 2*g + h; accumulator
        //      column rb holds j = 4*(rb % BQ) + rb / BQ
        constexpr int BQ = BN / 4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = i0 + 16 * warp + 2 * g + h;
            if (i >= p.I) continue;
            float* out = p.partial + ((long long)blockIdx.z * p.I + i) * p.J + j0;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int rb = 8 * j + 2 * t + c;
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

int tc_wg_bn(int J) { return J % 64 == 0 ? 64 : 32; }   // at most 64: 1.5 x BN fp32 accumulator registers per MMA thread

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
    CPB_REQUIRE(tc_offsets_fit(p.batch, p.big_img) && p.m_per_split < (1ll << 30) && p.Wo < 65536 && p.Ho * p.Wo < 65536,
                "tc_wgrad: tensor too large for 32-bit offsets");
    CPB_REQUIRE(p.passes == 3 || p.passes == 1, "tc_wgrad: passes must be 3 or 1, got %d", p.passes);
    if (p.passes == 1) return tc_wg_bn(p.J) == 64 ? tc_wg_launch<64, 1>(p, stream) : tc_wg_launch<32, 1>(p, stream);
    return tc_wg_bn(p.J) == 64 ? tc_wg_launch<64, 3>(p, stream) : tc_wg_launch<32, 3>(p, stream);
}

}  // namespace cpb
