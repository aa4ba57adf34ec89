// GAE (reference utils.py:45-50) on the device in float64: the single-rollout scan behind cpb_gae and learn(), and the
// segmented scan behind cpb_gae_segments and learn_segments().
#include "ppo.cuh"

namespace cpb {

namespace {

// ---------------------------------------------------------------------------------------------
// GAE: backward affine scan in float64, one CTA
// ---------------------------------------------------------------------------------------------
struct Affine { double a, b; };   // y -> a*y + b
__device__ __forceinline__ Affine compose(const Affine& first, const Affine& second) {
    return Affine{first.a * second.a, first.b * second.a + second.b};   // second(first(y))
}

constexpr int kGaeThreads = 1024;   // the scan's grouping (and so its rounding) depends on it: every GAE kernel uses it

// adv[0..T) of one rollout by the CTA's kGaeThreads threads: the reference's backward recursion as an affine scan.
// Ends with a barrier, so the CTA may read all of adv afterwards.
__device__ __forceinline__ void gae_scan(const double* __restrict__ rewards, const double* __restrict__ values,
                                         double bootstrap, const double* __restrict__ dones, int T, double gamma,
                                         double lam, double* __restrict__ adv) {
    __shared__ Affine warp_tot[32];
    __shared__ double carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double c = gamma * lam;
    if (tid == 0) carry_s = 0.0;
    __syncthreads();
    // u = reversed time index: y[u] = delta[u] + c*y[u-1]
    for (int base = 0; base < T; base += 1024) {
        const int u = base + tid;
        Affine f{1.0, 0.0};
        if (u < T) {
            const int t = T - 1 - u;
            const double vnext = t + 1 < T ? values[t + 1] : bootstrap;
            const double delta = rewards[t] + (1.0 - dones[t]) * gamma * vnext - values[t];
            f = Affine{c, delta};
        }
        // inclusive warp scan (composition order: earlier u first)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double pa = __shfl_up_sync(0xffffffffu, f.a, o);
            const double pb = __shfl_up_sync(0xffffffffu, f.b, o);
            if (lane >= o) f = compose(Affine{pa, pb}, f);
        }
        if (lane == 31) warp_tot[warp] = f;
        __syncthreads();
        if (warp == 0) {
            Affine g = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double pa = __shfl_up_sync(0xffffffffu, g.a, o);
                const double pb = __shfl_up_sync(0xffffffffu, g.b, o);
                if (lane >= o) g = compose(Affine{pa, pb}, g);
            }
            warp_tot[lane] = g;
        }
        __syncthreads();
        if (warp > 0) f = compose(warp_tot[warp - 1], f);
        const double carry = carry_s;
        const double y = f.a * carry + f.b;
        if (u < T) adv[T - 1 - u] = y;
        __syncthreads();
        if (tid == 1023) carry_s = y;
        __syncthreads();
    }
}

// returns = adv + values, advantages normalised by the mean and population std of adv[0..T) (numpy: mean, then mean of
// squared deviations), by the CTA's kGaeThreads threads; each output may be null
__device__ __forceinline__ void gae_normalise(const double* __restrict__ adv, const double* __restrict__ values, int T,
                                              double* __restrict__ ret_out, double* __restrict__ advn_out,
                                              float* __restrict__ ret32, float* __restrict__ advn32) {
    __shared__ double red[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double s = 0.0;
    for (int i = tid; i < T; i += 1024) s += adv[i];
    s = warp_sum(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (warp == 0) {
        double t = red[lane];
        t = warp_sum(t);
        if (lane == 0) red[0] = t;
    }
    __syncthreads();
    const double mean = red[0] / T;
    __syncthreads();
    double q = 0.0;
    for (int i = tid; i < T; i += 1024) { const double d = adv[i] - mean; q += d * d; }
    q = warp_sum(q);
    if (lane == 0) red[warp] = q;
    __syncthreads();
    if (warp == 0) {
        double t = red[lane];
        t = warp_sum(t);
        if (lane == 0) red[0] = t;
    }
    __syncthreads();
    const double sd = sqrt(red[0] / T);
    for (int i = tid; i < T; i += 1024) {
        const double a = adv[i];
        const double r = a + values[i];
        const double an = (a - mean) / (sd + 1e-8);
        if (ret_out != nullptr) ret_out[i] = r;
        if (advn_out != nullptr) advn_out[i] = an;
        if (ret32 != nullptr) ret32[i] = (float)r;
        if (advn32 != nullptr) advn32[i] = (float)an;
    }
}

__global__ void __launch_bounds__(kGaeThreads)
gae_kernel(const double* __restrict__ rewards, const double* __restrict__ values, double bootstrap,
           const double* __restrict__ dones, int T, double gamma, double lam, double* __restrict__ adv_out,
           double* __restrict__ ret_out, double* __restrict__ advn_out, float* __restrict__ ret32,
           float* __restrict__ advn32, double* __restrict__ scratch /* [T] when adv_out is null */) {
    double* adv = adv_out != nullptr ? adv_out : scratch;
    gae_scan(rewards, values, bootstrap, dones, T, gamma, lam, adv);
    gae_normalise(adv, values, T, ret_out, advn_out, ret32, advn32);
}

// Segmented GAE, step 1: CTA s scans rows [offsets[s], offsets[s+1]) with bootstrap[s] after its last row
__global__ void __launch_bounds__(kGaeThreads)
gae_segments_scan_kernel(const double* __restrict__ rewards, const double* __restrict__ values,
                         const double* __restrict__ bootstrap, const double* __restrict__ dones,
                         const int32_t* __restrict__ offsets, double gamma, double lam, double* __restrict__ adv) {
    const int s = blockIdx.x;
    const int begin = offsets[s], T = offsets[s + 1] - begin;
    gae_scan(rewards + begin, values + begin, bootstrap[s], dones + begin, T, gamma, lam, adv + begin);
}

// Segmented GAE, step 2: one normalisation over all rows of the update
__global__ void __launch_bounds__(kGaeThreads)
gae_normalise_kernel(const double* __restrict__ adv, const double* __restrict__ values, int rows,
                     double* __restrict__ ret_out, double* __restrict__ advn_out, float* __restrict__ ret32,
                     float* __restrict__ advn32) {
    gae_normalise(adv, values, rows, ret_out, advn_out, ret32, advn32);
}

}  // namespace

int32_t launch_gae(const double* rewards, const double* values, double bootstrap, const double* dones, int T, double gamma,
                   double lam, double* adv_out, double* ret_out, double* advn_out, float* ret32, float* advn32,
                   double* scratch, cudaStream_t s) {
    gae_kernel<<<1, kGaeThreads, 0, s>>>(rewards, values, bootstrap, dones, T, gamma, lam, adv_out, ret_out, advn_out, ret32,
                                         advn32, scratch);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t launch_gae_segments(const double* rewards, const double* values, const double* bootstrap, const double* dones,
                            const int32_t* offsets, int num_segments, int rows, double gamma, double lam, double* adv,
                            double* ret_out, double* advn_out, float* ret32, float* advn32, cudaStream_t s) {
    gae_segments_scan_kernel<<<num_segments, kGaeThreads, 0, s>>>(rewards, values, bootstrap, dones, offsets, gamma, lam, adv);
    CPB_LAUNCHED();
    gae_normalise_kernel<<<1, kGaeThreads, 0, s>>>(adv, values, rows, ret_out, advn_out, ret32, advn32);
    CPB_LAUNCHED();
    return CPB_OK;
}

}  // namespace cpb

using namespace cpb;

extern "C" {

int32_t cpb_gae(const double* rewards, const double* values, double bootstrap_value, const double* dones, int32_t T,
                double gamma, double lam, double* advantages, double* returns, double* advantages_norm, void* stream) {
    CPB_REQUIRE(rewards && values && dones && T >= 1, "gae: bad arguments");
    CPB_REQUIRE(advantages != nullptr, "gae: advantages output is required");
    return launch_gae(rewards, values, bootstrap_value, dones, T, gamma, lam, advantages, returns, advantages_norm, nullptr,
                      nullptr, nullptr, (cudaStream_t)stream);
}

int32_t cpb_gae_segments(const double* rewards, const double* values, const double* bootstrap_values, const double* dones,
                         const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma, double lam,
                         double* advantages, double* returns, double* advantages_norm, void* stream) {
    CPB_REQUIRE(num_segments >= 1 && rows >= num_segments, "gae_segments: need 1 <= num_segments <= rows");
    CPB_REQUIRE(rewards && values && bootstrap_values && dones && segment_offsets, "gae_segments: NULL pointer");
    CPB_REQUIRE(advantages != nullptr, "gae_segments: advantages output is required");
    return launch_gae_segments(rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                               advantages, returns, advantages_norm, nullptr, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
