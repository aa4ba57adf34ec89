// Running normalisation of the PPO's observations and rewards (Stable-Baselines3's VecNormalize) on the device.
//
// Statistics are RunningMeanStd(epsilon=1e-4) in float64: a device double[2*dim + 1] = [mean | var | count].  A batch of
// n rows is reduced two-pass (the mean, then sum (x - mean)^2, ddof 0) and merged with Chan's formula, written with
// explicit round-to-nearest operations so that no contraction changes it:
//   delta = mu_b - mu,  t = c + n,  mu' = mu + delta*n/t,  var' = (var*c + var_b*n + delta^2*c*n/t)/t,  c' = t.
//
// obs_norm_kernel: one CTA per 32-column tile (a cluster of up to 8 CTAs walks the tiles), 16 row groups per tile.  A
// column's sums depend only on (B, D): rows r = ty, ty + 16, ... in order per thread, then the 16 partials in ty order.
// Rows are never split across CTAs, so no cross-CTA reduction is needed; the only shared value is the count, which every
// CTA reads before a cluster barrier and the cluster's rank 0 replaces after it.
#include <cmath>

#include "common.cuh"

namespace cpb {

constexpr int kNormTileCols = 32, kNormRowGroups = 16, kNormMaxCluster = 8, kRewardThreads = 256;

__device__ __forceinline__ void merge_moments(double& mean, double& var, double count, double bmean, double bvar, double n) {
    const double delta = __dsub_rn(bmean, mean), tot = __dadd_rn(count, n);
    mean = __dadd_rn(mean, __ddiv_rn(__dmul_rn(delta, n), tot));
    const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(var, count), __dmul_rn(bvar, n)),
                                __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(delta, delta), count), n), tot));
    var = __ddiv_rn(m2, tot);
}

// clip(x / sqrt(var + eps), -clip, clip) in float64, rounded once to fp32
__device__ __forceinline__ float scaled_clip(double x, double var, double eps, double clip) {
    const double y = __ddiv_rn(x, __dsqrt_rn(__dadd_rn(var, eps)));
    return (float)fmin(fmax(y, -clip), clip);
}

struct ObsNormArgs {
    const float* a;      // columns [0, za) of row r: a[r * za + c]
    const float* b;      // columns [za, D) of row r: b[r * mb + c - za] (mb = D - za)
    int za, mb, batch;
    double* stats;       // [mean | var | count]
    int update;
    double clip, eps;
    float* out;          // [B, D]
};

__device__ __forceinline__ float obs_at(const ObsNormArgs& p, int r, int c) {
    return c < p.za ? __ldg(p.a + (int64_t)r * p.za + c) : __ldg(p.b + (int64_t)r * p.mb + (c - p.za));
}

// the sum of one column's 16 row-group partials in ty order, returned to every thread of the column
__device__ __forceinline__ double column_total(double v, double (*part)[kNormTileCols + 1]) {
    __syncthreads();                  // part may still be read by a previous call
    part[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kNormRowGroups; ++k) s = __dadd_rn(s, part[k][threadIdx.x]);
    return s;
}

__global__ void __launch_bounds__(kNormTileCols * kNormRowGroups) obs_norm_kernel(const ObsNormArgs p) {
    __shared__ double part[kNormRowGroups][kNormTileCols + 1];
    const int D = p.za + p.mb, B = p.batch, tx = threadIdx.x, ty = threadIdx.y;
    const double count = p.stats[2 * D], n = (double)B;
    // every CTA has read the count before rank 0 of the cluster replaces it
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    for (int c0 = blockIdx.x * kNormTileCols; c0 < D; c0 += gridDim.x * kNormTileCols) {
        const int c = c0 + tx;
        const bool col = c < D;
        double mean = col ? p.stats[c] : 0.0, var = col ? p.stats[D + c] : 1.0;
        if (p.update) {
            double s = 0.0;
            if (col)
                for (int r = ty; r < B; r += kNormRowGroups) s = __dadd_rn(s, (double)obs_at(p, r, c));
            const double bmean = __ddiv_rn(column_total(s, part), n);
            double q = 0.0;
            if (col)
                for (int r = ty; r < B; r += kNormRowGroups) {
                    const double d = __dsub_rn((double)obs_at(p, r, c), bmean);
                    q = __dadd_rn(q, __dmul_rn(d, d));
                }
            const double bvar = __ddiv_rn(column_total(q, part), n);
            merge_moments(mean, var, count, bmean, bvar, n);
            if (col && ty == 0) {
                p.stats[c] = mean;
                p.stats[D + c] = var;
            }
        }
        if (col)
            for (int r = ty; r < B; r += kNormRowGroups)
                p.out[(int64_t)r * D + c] = scaled_clip(__dsub_rn((double)obs_at(p, r, c), mean), var, p.eps, p.clip);
    }
    if (p.update && blockIdx.x == 0 && tx == 0 && ty == 0) p.stats[2 * D] = __dadd_rn(count, n);
}

// RunningMeanStd(epsilon=1e-4)'s initial state: mean 0, var 1, count 1e-4
__global__ void running_norm_init_kernel(double* stats, int D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= 2 * D) stats[i] = i < D ? 0.0 : (i < 2 * D ? 1.0 : 1e-4);
}

int32_t launch_obs_norm(const ObsNormArgs& p, cudaStream_t stream) {
    const int tiles = cdiv(p.za + p.mb, kNormTileCols);
    const unsigned grid = (unsigned)(tiles < kNormMaxCluster ? tiles : kNormMaxCluster);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kNormTileCols, kNormRowGroups);
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = grid; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    CPB_CUDA(cudaLaunchKernelEx(&cfg, obs_norm_kernel, p));
    CPB_LAUNCHED();
    return CPB_OK;
}

// sum of v over the CTA's threads in a fixed order, returned to every thread; red: shared [kRewardThreads / 32]
__device__ __forceinline__ double block_total(double v, double* red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kRewardThreads / 32; ++w) s = __dadd_rn(s, red[w]);
    return s;
}

struct RewardNormArgs {
    double* stats;             // [mean | var | count] of the returns
    double* ret;               // [num_envs]
    const int32_t* env_ids;    // [B], clamped into [0, num_envs)
    const float* rewards;      // [B]
    const int32_t* dones;      // [B], nonzero = terminal
    int batch, num_envs;
    double gamma, clip, eps;
    float* out;                // [B]
};

__device__ __forceinline__ int env_of(const RewardNormArgs& p, int i) {
    const int e = p.env_ids[i];
    return e < 0 ? 0 : (e >= p.num_envs ? p.num_envs - 1 : e);
}

// VecNormalize.step_wait's reward path for the stepped environments, in one CTA:
// ret = ret * gamma + r; update the return statistics with ret[stepped]; r' = clip(r / sqrt(var + eps)); ret = 0 if done
__global__ void __launch_bounds__(kRewardThreads) reward_norm_kernel(const RewardNormArgs p) {
    __shared__ double red[kRewardThreads / 32];
    const int B = p.batch;
    for (int i = threadIdx.x; i < B; i += kRewardThreads) {
        const int e = env_of(p, i);
        p.ret[e] = __dadd_rn(__dmul_rn(p.ret[e], p.gamma), (double)p.rewards[i]);
    }
    __syncthreads();
    double s = 0.0;
    for (int i = threadIdx.x; i < B; i += kRewardThreads) s = __dadd_rn(s, p.ret[env_of(p, i)]);
    const double n = (double)B, bmean = __ddiv_rn(block_total(s, red), n);
    double q = 0.0;
    for (int i = threadIdx.x; i < B; i += kRewardThreads) {
        const double d = __dsub_rn(p.ret[env_of(p, i)], bmean);
        q = __dadd_rn(q, __dmul_rn(d, d));
    }
    const double bvar = __ddiv_rn(block_total(q, red), n);
    double mean = p.stats[0], var = p.stats[1];
    const double count = p.stats[2];
    merge_moments(mean, var, count, bmean, bvar, n);
    __syncthreads();                  // every thread has read the statistics and ret before they change
    if (threadIdx.x == 0) {
        p.stats[0] = mean;
        p.stats[1] = var;
        p.stats[2] = __dadd_rn(count, n);
    }
    for (int i = threadIdx.x; i < B; i += kRewardThreads) {
        p.out[i] = scaled_clip((double)p.rewards[i], var, p.eps, p.clip);
        if (p.dones[i]) p.ret[env_of(p, i)] = 0.0;
    }
}

int32_t launch_reward_norm(const RewardNormArgs& p, cudaStream_t stream) {
    reward_norm_kernel<<<1, kRewardThreads, 0, stream>>>(p);
    CPB_LAUNCHED();
    return CPB_OK;
}

static int32_t check_norm_config(const cpb_running_norm* cfg, const char* who) {
    CPB_REQUIRE(cfg != nullptr, "%s: NULL config", who);
    CPB_REQUIRE(cfg->dim >= 1, "%s: dim must be >= 1, got %d", who, cfg->dim);
    CPB_REQUIRE(std::isfinite(cfg->clip) && cfg->clip > 0.f, "%s: clip must be finite and > 0", who);
    CPB_REQUIRE(std::isfinite(cfg->epsilon) && cfg->epsilon > 0.0, "%s: epsilon must be finite and > 0", who);
    return CPB_OK;
}

static int32_t check_reward_args(const cpb_running_norm* cfg, const double* ret_stats, const double* returns,
                                 const int32_t* env_ids, const float* rewards, const int32_t* dones, int32_t batch,
                                 int32_t num_envs, double gamma, const float* out) {
    CPB_TRY(check_norm_config(cfg, "reward normalisation"));
    CPB_REQUIRE(cfg->dim == 1, "reward normalisation: dim must be 1, got %d", cfg->dim);
    CPB_REQUIRE(ret_stats && returns && env_ids && rewards && dones && out, "reward normalisation: NULL pointer");
    CPB_REQUIRE(batch >= 1 && num_envs >= 1, "reward normalisation: batch %d and num_envs %d must be >= 1", batch, num_envs);
    CPB_REQUIRE(gamma >= 0.0 && gamma <= 1.0, "reward normalisation: gamma must lie in [0, 1]");
    return CPB_OK;
}

static RewardNormArgs reward_args(const cpb_running_norm* cfg, double* ret_stats, double* returns, const int32_t* env_ids,
                                  const float* rewards, const int32_t* dones, int32_t batch, int32_t num_envs,
                                  double gamma, float* out) {
    return RewardNormArgs{ret_stats, returns, env_ids, rewards, dones, batch, num_envs, gamma, (double)cfg->clip,
                          cfg->epsilon, out};
}

// The normalisation half of an actor call (actor.cu's encode_predict): checked before anything is enqueued, then the
// normalised state assembly in place of the plain one, and the reward kernel when rewards are given.
int32_t check_actor_norm(const cpb_actor_norm* n, int32_t state_dim, int32_t batch) {
    CPB_REQUIRE(n != nullptr, "actor normalisation: NULL cpb_actor_norm");
    CPB_TRY(check_norm_config(&n->obs, "observation normalisation"));
    CPB_REQUIRE(n->obs.dim == state_dim, "observation normalisation: dim %d != the PPO's state_dim %d", n->obs.dim, state_dim);
    CPB_REQUIRE(n->obs_stats != nullptr, "observation normalisation: NULL statistics");
    if (n->rewards != nullptr)
        CPB_TRY(check_reward_args(&n->reward, n->ret_stats, n->returns, n->env_ids, n->rewards, n->dones, batch,
                                  n->num_envs, n->gamma, n->rewards_out));
    return CPB_OK;
}

int32_t launch_actor_obs_norm(const cpb_actor_norm* n, const float* latent, int z, const float* meas, int m, int batch,
                              float* state, cudaStream_t stream) {
    return launch_obs_norm(ObsNormArgs{latent, meas, z, m, batch, n->obs_stats, n->update != 0, (double)n->obs.clip,
                                       n->obs.epsilon, state}, stream);
}

int32_t launch_actor_reward_norm(const cpb_actor_norm* n, int batch, cudaStream_t stream) {
    if (n->rewards == nullptr) return CPB_OK;
    return launch_reward_norm(reward_args(&n->reward, n->ret_stats, n->returns, n->env_ids, n->rewards, n->dones, batch,
                                          n->num_envs, n->gamma, n->rewards_out), stream);
}

}  // namespace cpb

using namespace cpb;

int32_t cpb_running_norm_init(const cpb_running_norm* cfg, double* stats, void* stream) {
    CPB_TRY(check_norm_config(cfg, "cpb_running_norm_init"));
    CPB_REQUIRE(stats != nullptr, "cpb_running_norm_init: NULL statistics");
    const int D = cfg->dim;
    running_norm_init_kernel<<<cdiv(2 * D + 1, 256), 256, 0, (cudaStream_t)stream>>>(stats, D);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t cpb_obs_normalize(const cpb_running_norm* cfg, double* stats, const float* x, int32_t batch, int32_t update,
                          float* out, void* stream) {
    CPB_TRY(check_norm_config(cfg, "cpb_obs_normalize"));
    CPB_REQUIRE(stats && x && out, "cpb_obs_normalize: NULL pointer");
    CPB_REQUIRE(batch >= 1, "cpb_obs_normalize: batch must be >= 1, got %d", batch);
    return launch_obs_norm(ObsNormArgs{x, nullptr, cfg->dim, 0, batch, stats, update != 0, (double)cfg->clip, cfg->epsilon,
                                       out}, (cudaStream_t)stream);
}

int32_t cpb_reward_normalize(const cpb_running_norm* cfg, double* ret_stats, double* returns, const int32_t* env_ids,
                             const float* rewards, const int32_t* dones, int32_t batch, int32_t num_envs, double gamma,
                             float* out, void* stream) {
    CPB_TRY(check_reward_args(cfg, ret_stats, returns, env_ids, rewards, dones, batch, num_envs, gamma, out));
    return launch_reward_norm(reward_args(cfg, ret_stats, returns, env_ids, rewards, dones, batch, num_envs, gamma, out),
                              (cudaStream_t)stream);
}
