// The opt-in (CPB_PPO_PERSISTENT=1) persistent learn() kernel, reached only through learn_persistent (see ppo.cuh).
#include <cooperative_groups.h>

#include <cstdlib>

#include "elementwise.cuh"
#include "ppo_device.cuh"

namespace cpb {

namespace {

// ---------------------------------------------------------------------------------------------
// The driver's whole update block as ONE persistent cooperative kernel (train.py:171-207 after GAE / theta_old):
// num_epochs x ceil(T / batch) minibatch steps, each = forward (one phase per layer index, both trunks) -> head + loss ->
// backward (one phase per layer index, top down) -> TF-Adam, with grid-wide barriers between the dependent phases instead
// of ~2 D + 5 kernel launches per minibatch (D = the deeper trunk's depth; ~330 launches of 5-30 us kernels per learn()
// at the default two layers per trunk).  One CTA per SM, 2 independent groups of 128 threads per CTA;
// a phase's 32x32 output tiles are dealt round-robin to the 4 x gridDim groups; the arithmetic per tile is the
// stand-alone small_gemm_kernel's (same gemm_tile), so the results are those of the launch-per-kernel path up to the
// order in which the per-CTA loss partials are summed.
// ---------------------------------------------------------------------------------------------
struct LearnArgs {
    cpb_ppo_spec spec;
    PpoLayout L;
    PpoPlan pl;
    float* params; float* grads; float* adam_m; float* adam_v; float* adam_powers;
    const float* lr_dev;
    const float* states; const float* actions;
    const int32_t* perms;
    float* metrics;
    int T, batch_size, num_epochs, nmb;
    Guards gd;             // gd.stop == nullptr: no guards, 5-wide metrics rows
    HeadShape hs;          // read by the categorical instantiation only
};
// a __grid_constant__ kernel parameter: within the 4 KB parameter space at every architecture (8 layers per trunk)
static_assert(sizeof(LearnArgs) <= 4096, "LearnArgs exceeds the kernel parameter space");

constexpr int kGroupsPerCta = 2;
constexpr int kLearnThreads = kGroupsPerCta * kTileThreads;
constexpr size_t kLearnSmem = (size_t)kGroupsPerCta * 2 * 2 * TK * (TS + 4) * sizeof(float);

__device__ __forceinline__ int tiles_of(int n) { return (n + TS - 1) / TS; }

template <int GATHER>
__device__ __forceinline__ void run_phase(const GemmJob* jobs, int njobs, float* smem, int gid, int ngroups) {
    const int group = threadIdx.x / kTileThreads, gtid = threadIdx.x % kTileThreads;
    float (*As)[TK][TS + 4] = reinterpret_cast<float (*)[TK][TS + 4]>(smem + (size_t)group * 2 * 2 * TK * (TS + 4));
    float (*Bs)[TK][TS + 4] = As + 2;
    int total = 0;
    for (int j = 0; j < njobs; ++j) total += tiles_of(jobs[j].M) * tiles_of(jobs[j].N);
    for (int t = gid; t < total; t += ngroups) {
        int j = 0, r = t;
        for (;; ++j) {
            const int nt = tiles_of(jobs[j].M) * tiles_of(jobs[j].N);
            if (r < nt) break;
            r -= nt;
        }
        const int mt = tiles_of(jobs[j].M);
        const int mi = r % mt, ni = r / mt;
        gemm_tile<GATHER>(jobs[j], mi * TS, ni * TS, mi == 0, gtid, As, Bs,
                          [group] { asm volatile("bar.sync %0, 128;" ::"r"(group + 1) : "memory"); });
    }
}

template <int CAT>
__global__ void __launch_bounds__(kLearnThreads, 1)
ppo_learn_persistent_kernel(const __grid_constant__ LearnArgs a) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    extern __shared__ __align__(16) float learn_smem[];
    __shared__ float red[8][8];
    __shared__ float tot[8];
    __shared__ float nred[kLearnThreads / 32];
    const cpb_ppo_spec& sp = a.spec;
    const cpb_ppo_config& c = sp.base;
    const PpoLayout& L = a.L;
    const PpoPlan& pl = a.pl;
    const Guards& gd = a.gd;
    const int A = c.num_actions, D = max_depth(sp);
    const int ngroups = gridDim.x * kGroupsPerCta;
    const int gid = blockIdx.x * kGroupsPerCta + threadIdx.x / kTileThreads;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mcols = gd.stop != nullptr ? 7 : 5;
    float* params = a.params;
    float* grads = a.grads;

    // Every CTA runs every minibatch and reaches every grid.sync: the layer loops run to the same D in every CTA, and the
    // guards only predicate the Adam step, on values every CTA reads after a grid.sync (the stop word ppo_finalize wrote
    // two barriers earlier, the norm partials of all CTAs).
    for (int e = 0; e < a.num_epochs; ++e)
        for (int i = 0; i < a.nmb; ++i) {
            const int begin = i * a.batch_size;
            const int B = begin + a.batch_size <= a.T ? a.batch_size : a.T - begin;
            const int32_t* idx = a.perms + (long long)e * a.T + begin;
            float* mt = a.metrics ? a.metrics + ((long long)e * a.nmb + i) * mcols : nullptr;
            GemmJob jobs[6];
            // ---- forward: layer l of both trunks per phase
            for (int l = 0; l < D; ++l) {
                const int n = trunk_fwd_jobs(sp, L, pl, params, a.states, idx, B, l, jobs);
                if (l == 0) run_phase<1>(jobs, n, learn_smem, gid, ngroups);
                else run_phase<0>(jobs, n, learn_smem, gid, ngroups);
                grid.sync();
            }
            // ---- head: one warp per sample, per-CTA partial loss sums
            {
                HeadArgs h = head_args(sp, a.hs, L, params, B);
                h.hp = trunk_buf(pl.h, sp, 0, sp.num_policy - 1, B); h.hv = trunk_buf(pl.h, sp, 1, sp.num_value - 1, B);
                h.actions = a.actions; h.returns = pl.ret32; h.adv = pl.adv32; h.idx = idx;
                h.logp_old_in = pl.logp_old; h.logp_old_gathered = 1;
                h.dpre = pl.dpre; h.dv = pl.dv; h.partial = pl.partial;
                h.dhp = trunk_buf(pl.dh, sp, 0, sp.num_policy - 1, B); h.dhv = trunk_buf(pl.dh, sp, 1, sp.num_value - 1, B);
                h.kl_term = gd.stop != nullptr;
                float vals[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                for (int b = blockIdx.x * 8 + warp; b < B; b += gridDim.x * 8) head_row<1, CAT>(h, b, lane, vals);
                head_block_reduce(vals, red, pl.partial + blockIdx.x * 8);
            }
            grid.sync();
            // ---- loss metrics + logstd gradient (CTA 0), then the backward pass top down: layer l of both trunks per
            // phase, the head weight gradients with the top layer (their own tile list when that layer gathers the states)
            if (blockIdx.x == 0)
                ppo_finalize<CAT>(pl.partial, gridDim.x, B, A, params + L.off[L.logstd()], c.value_scale, c.entropy_scale,
                                  grads + L.off[L.logstd()], mt, tot, gd);
            for (int l = D - 1; l >= 0; --l) {
                int n = trunk_bwd_jobs(sp, L, pl, params, grads, a.states, idx, B, l, jobs);
                if (l > 0) {
                    if (l == D - 1) { head_bwd_jobs(sp, L, pl, grads, B, CAT ? a.hs.N : sp.base.num_actions, jobs + n); n += 2; }
                    run_phase<0>(jobs, n, learn_smem, gid, ngroups);
                } else {
                    run_phase<2>(jobs, n, learn_smem, gid, ngroups);
                    if (D == 1) {
                        head_bwd_jobs(sp, L, pl, grads, B, CAT ? a.hs.N : sp.base.num_actions, jobs);
                        run_phase<0>(jobs, 2, learn_smem, gid, ngroups);
                    }
                }
                grid.sync();
            }
            // ---- guards: per-CTA sums of g^2, a barrier, then the same fixed-order sum of all partials in every CTA
            float gscale = 1.f;
            bool apply = true;
            if (gd.stop != nullptr) {
                const long long n4 = L.total / 4;
                const float s = block_sum(sumsq_share(reinterpret_cast<const float4*>(grads), n4,
                                                      (long long)blockIdx.x * blockDim.x + threadIdx.x,
                                                      (long long)gridDim.x * blockDim.x), nred);
                if (threadIdx.x == 0) gd.norm_partial[blockIdx.x] = s;
                grid.sync();
                float t = 0.f;
                for (int k = threadIdx.x; k < (int)gridDim.x; k += blockDim.x) t += __ldcg(gd.norm_partial + k);
                t = block_sum(t, nred);
                gscale = clip_coefficient(t, gd.max_norm);
                const uint32_t stop = __ldcg(gd.stop);
                apply = stop == 0u;
                if (blockIdx.x == 0 && threadIdx.x == 0 && mt != nullptr && stop != 2u) mt[6] = sqrtf(t);
            }
            // ---- TF ApplyAdam (adam_update, as in adam_kernel), beta powers advanced after the barrier
            if (apply) {
                const float lr_t = a.lr_dev[0];
                const float p0 = __ldcg(a.adam_powers), p1 = __ldcg(a.adam_powers + 1);
                const float alpha = lr_t * sqrtf(1.f - p1) / (1.f - p0);
                const float beta1 = 0.9f, beta2 = 0.999f, epsilon = 1e-8f;
                const float omb1 = 1.f - beta1, omb2 = 1.f - beta2;
                const long long n4 = L.total / 4;
                float4* p4 = reinterpret_cast<float4*>(params);
                const float4* g4 = reinterpret_cast<const float4*>(grads);
                float4* m4 = reinterpret_cast<float4*>(a.adam_m);
                float4* v4 = reinterpret_cast<float4*>(a.adam_v);
                for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += (long long)gridDim.x * blockDim.x) {
                    float4 gv = __ldcg(g4 + k);
                    if (gd.stop != nullptr) { gv.x *= gscale; gv.y *= gscale; gv.z *= gscale; gv.w *= gscale; }
                    float4 mv = m4[k], vv = v4[k], pv = p4[k];
                    adam_update(gv, mv, vv, pv, alpha, omb1, omb2, epsilon);
                    m4[k] = mv; v4[k] = vv; p4[k] = pv;
                }
            }
            grid.sync();
            if (blockIdx.x == 0 && threadIdx.x == 0 && apply) {
                a.adam_powers[0] *= 0.9f; a.adam_powers[1] *= 0.999f;
                if (gd.steps != nullptr) gd.steps[0] += 1;
            }
        }
}

int g_learn_grid = 0;      // co-resident CTAs of the persistent kernel (0: not initialised, -1: unavailable)

int32_t learn_persistent_init() {
    if (g_learn_grid != 0) return CPB_OK;
    int dev = 0, sms = 0, coop = 0, per_sm = 0;
    CPB_CUDA(cudaGetDevice(&dev));
    CPB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CPB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    int per_sm_cat = 0;     // the categorical instantiation shares the grid
    CPB_CUDA(cudaFuncSetAttribute(ppo_learn_persistent_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLearnSmem));
    CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ppo_learn_persistent_kernel<0>, kLearnThreads, kLearnSmem));
    CPB_CUDA(cudaFuncSetAttribute(ppo_learn_persistent_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLearnSmem));
    CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_cat, ppo_learn_persistent_kernel<1>, kLearnThreads, kLearnSmem));
    if (per_sm_cat < per_sm) per_sm = per_sm_cat;
    // Opt-in (CPB_PPO_PERSISTENT=1): slower than the launch-per-kernel path -- the 32x32 / 64-thread gemm_tile is latency-bound
    // (8 dependent global round trips per K = 500 tile) and one CTA per SM leaves 8 warps to hide them, where the stand-alone
    // kernels run ~16 CTAs per SM; the barriers are not the cost.  Kept because it is parity-green (tests run both paths) and is the skeleton for a tile routine that
    // stages a whole K strip per barrier phase.
    const char* e = getenv("CPB_PPO_PERSISTENT");
    const bool want = e != nullptr && atoi(e) != 0;
    g_learn_grid = (coop && per_sm >= 1 && want) ? (sms < kMaxPersistentCtas ? sms : kMaxPersistentCtas) : -1;
    return CPB_OK;
}

}  // namespace

int32_t learn_persistent(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, float* params,
                         float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                         const float* states, const float* actions, int T, int num_epochs, int batch_size, int nmb,
                         const int32_t* perms, float* metrics, const Guards& gd, cudaStream_t s, bool* launched) {
    *launched = false;
    CPB_TRY(learn_persistent_init());
    if (g_learn_grid <= 0 || num_epochs <= 0) return CPB_OK;
    // all minibatch steps in ONE cooperative launch
    LearnArgs a;
    memset(&a, 0, sizeof(a));
    a.spec = *sp; a.L = L; a.pl = pl;
    a.params = params; a.grads = grads; a.adam_m = adam_m; a.adam_v = adam_v; a.adam_powers = adam_powers; a.lr_dev = lr_dev;
    a.states = states; a.actions = actions; a.perms = perms; a.metrics = metrics;
    a.T = T; a.batch_size = batch_size; a.num_epochs = num_epochs; a.nmb = nmb;
    a.gd = gd;
    a.hs = hs;
    void* args[] = {&a};
    void* kernel = hs.cat ? (void*)ppo_learn_persistent_kernel<1> : (void*)ppo_learn_persistent_kernel<0>;
    CPB_CUDA(cudaLaunchCooperativeKernel(kernel, dim3((unsigned)g_learn_grid), dim3(kLearnThreads), args, kLearnSmem, s));
    CPB_LAUNCHED();
    *launched = true;
    return CPB_OK;
}

}  // namespace cpb
