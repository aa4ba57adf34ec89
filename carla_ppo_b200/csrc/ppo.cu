// PPO update path behind the C ABI: Gaussian-policy / value MLPs (reference ppo.py:38-66), clipped
// surrogate + value + entropy loss and its gradient (ppo.py:119-144), GAE (utils.py:45-50) and the
// driver's update block (train.py:171-207).  Everything here is latency-bound (369 505 parameters,
// minibatches of a few hundred rows): the kernels are small bounds-checked fp32 tile GEMMs, batched
// over the two trunks (policy / value) so one minibatch step is ~11 launches with no host sync.
#include <cooperative_groups.h>

#include <cmath>

#include "common.cuh"
#include "elementwise.cuh"

namespace cpb {

namespace {

constexpr int kMaxPpoDepth = 8;                          // hidden layers per trunk (cpb_ppo_spec)
constexpr int kMaxPpoTensors = 4 * kMaxPpoDepth + 5;
constexpr int kLegacyPpoTensors = 13;                     // two layers per trunk (cpb_ppo_config)

// Hidden-layer count and widths of trunk t (0: policy, 1: value) of a checked spec
__host__ __device__ __forceinline__ int trunk_depth(const cpb_ppo_spec& sp, int t) { return t ? sp.num_value : sp.num_policy; }
__host__ __device__ __forceinline__ int trunk_width(const cpb_ppo_spec& sp, int t, int l) {
    return t ? sp.value_sizes[l] : sp.policy_sizes[l];
}
// width of layer l's input: the state for layer 0
__host__ __device__ __forceinline__ int trunk_in(const cpb_ppo_spec& sp, int t, int l) {
    return l ? trunk_width(sp, t, l - 1) : sp.base.state_dim;
}
__host__ __device__ __forceinline__ int trunk_last(const cpb_ppo_spec& sp, int t) { return trunk_width(sp, t, trunk_depth(sp, t) - 1); }
__host__ __device__ __forceinline__ int max_depth(const cpb_ppo_spec& sp) {
    return sp.num_policy > sp.num_value ? sp.num_policy : sp.num_value;
}

// Tensors in TF creation order (ppo.py:38-66): policy layer l {kernel, bias} at 2l, the action head {action_mean/kernel,
// action_mean/bias, action_logstd} at 2P, value layer l at 2P + 3 + 2l, value/{kernel, bias} last.  Dense layers are
// named dense, dense_1, ... across both trunks in that order.
struct PpoLayout {
    int np, nv, n;
    int64_t off[kMaxPpoTensors], size[kMaxPpoTensors];
    int32_t shape[kMaxPpoTensors][2];
    int64_t total;
    __host__ __device__ int w(int t, int l) const { return t ? 2 * np + 3 + 2 * l : 2 * l; }
    __host__ __device__ int b(int t, int l) const { return w(t, l) + 1; }
    __host__ __device__ int wm() const { return 2 * np; }
    __host__ __device__ int bm() const { return 2 * np + 1; }
    __host__ __device__ int logstd() const { return 2 * np + 2; }
    __host__ __device__ int wv() const { return 2 * np + 3 + 2 * nv; }
    __host__ __device__ int bv() const { return wv() + 1; }
};

// The policy head of a plan.  Gaussian (cat == 0): N = K = num_actions columns of action_mean and an action_logstd.
// Categorical (cpb_ppo_cat_spec, cat == 1): N = sum n_k logits in action_logits, component k's at columns
// [off[k], off[k+1]); its layout keeps the logstd slot at size 0, so both kinds share PpoLayout's indexing.
constexpr int kMaxLogits = 64;
struct HeadShape {
    int cat, K, N;
    int off[5];
};

HeadShape gauss_head(const cpb_ppo_spec* sp) {
    HeadShape hs;
    memset(&hs, 0, sizeof(hs));
    hs.K = hs.N = sp->base.num_actions;
    return hs;
}

PpoLayout make_ppo_layout(const cpb_ppo_spec* sp, const HeadShape& hs) {
    PpoLayout L;
    memset(&L, 0, sizeof(L));
    const int A = sp->base.num_actions;
    L.np = sp->num_policy; L.nv = sp->num_value; L.n = 2 * (L.np + L.nv) + 5;
    auto set = [&](int i, int rows, int cols) { L.shape[i][0] = rows; L.shape[i][1] = cols; };
    for (int t = 0; t < 2; ++t)
        for (int l = 0; l < trunk_depth(*sp, t); ++l) {
            set(L.w(t, l), trunk_in(*sp, t, l), trunk_width(*sp, t, l));
            set(L.b(t, l), trunk_width(*sp, t, l), 0);
        }
    if (hs.cat) { set(L.wm(), trunk_last(*sp, 0), hs.N); set(L.bm(), hs.N, 0); }
    else { set(L.wm(), trunk_last(*sp, 0), A); set(L.bm(), A, 0); set(L.logstd(), A, 0); }
    set(L.wv(), trunk_last(*sp, 1), 1); set(L.bv(), 1, 0);
    int64_t o = 0;
    for (int i = 0; i < L.n; ++i) {
        L.size[i] = (int64_t)L.shape[i][0] * (L.shape[i][1] ? L.shape[i][1] : 1);
        L.off[i] = o;
        o += align_up(L.size[i], 64);
    }
    L.total = o;
    return L;
}

// A categorical layout has no action_logstd: its public index i is PpoLayout's index i, or i + 1 past the head
__host__ __device__ __forceinline__ int cat_internal_index(const cpb_ppo_spec& sp, int i) { return i < 2 * sp.num_policy + 2 ? i : i + 1; }

const char* ppo_tensor_name(const cpb_ppo_spec* sp, int i) {
    static char dense[2 * kMaxPpoDepth][2][24];
    static const bool ready = [] {
        for (int k = 0; k < 2 * kMaxPpoDepth; ++k)
            for (int b = 0; b < 2; ++b) {
                char suffix[8] = "";
                if (k) snprintf(suffix, sizeof(suffix), "_%d", k);
                snprintf(dense[k][b], sizeof(dense[k][b]), "dense%s/%s", suffix, b ? "bias" : "kernel");
            }
        return true;
    }();
    (void)ready;
    static const char* heads[5] = {"action_mean/kernel", "action_mean/bias", "action_logstd", "value/kernel", "value/bias"};
    const int P = sp->num_policy, V = sp->num_value;
    if (i < 0 || i >= 2 * (P + V) + 5) return nullptr;
    if (i < 2 * P) return dense[i / 2][i % 2];
    if (i < 2 * P + 3) return heads[i - 2 * P];
    if (i < 2 * P + 3 + 2 * V) return dense[P + (i - 2 * P - 3) / 2][(i - 2 * P - 3) % 2];
    return heads[3 + i - (2 * P + 3 + 2 * V)];
}

// ---------------------------------------------------------------------------------------------
// small tile GEMM: C[M,N] (+)= A'[M,K] * B'[K,N], 32x32 tile, 128 threads, 2x4 per thread
// ---------------------------------------------------------------------------------------------
constexpr int TS = 32;   // tile edge
constexpr int TK = 64;   // reduction chunk (one global round trip per chunk: keep the chunk count low)

// operand access descriptors (element (o, r) = output index o, reduction index r)
struct Operand {
    const float* p;
    long long so, sr;       // strides for the output / reduction index
    const int32_t* gather;  // optional row gather applied to whichever index has the larger stride
    int gather_on_o;        // 1: gather indexes o, 0: gather indexes r
};

// GATHER: 0 = none, 1 = the A operand's output index goes through `gather`, 2 = its reduction index does.
// Compile-time so that the 16 loads of a chunk stay independent (a run-time check serialised them: each
// value load waited on a predicated index load that reused the same register).
template <int GATHER>
__device__ __forceinline__ long long a_offset(const Operand& a, int o, int r) {
    if (GATHER == 1) return (long long)__ldg(a.gather + o) * a.so + (long long)r * a.sr;      // the index vectors are launch inputs
    if (GATHER == 2) return (long long)o * a.so + (long long)__ldg(a.gather + r) * a.sr;
    return (long long)o * a.so + (long long)r * a.sr;
}

struct GemmJob {
    Operand a, b;            // a: (m, r), b: (n, r)
    int M, N, R;
    float* c;                // [M, ldc]
    int ldc;
    const float* bias;       // [N] or null
    const float* mask;       // [M, ldc] or null: out *= mask > 0
    int relu;
    float* colsum;           // [N] or null: colsum[n] = sum_r b(n, r)   (bias gradient; blockIdx.x == 0 only)
};

struct GemmBatch {
    GemmJob job[6];       // independent GEMMs of one launch (blockIdx.z); all with the same gather mode
};

// One 32x32 output tile of job J by a GROUP of kTileThreads = 128 threads (tid = 0..127), 2x4 outputs per thread.  `sync()` is
// the group's barrier: __syncthreads in the stand-alone kernel (one group per CTA), a named barrier in the persistent learn()
// kernel (two groups per CTA).  As / Bs: the group's double-buffered operand tiles [2][TK][TS + 4].
// (Round 1 used 64 threads with 4x4 outputs: 1024 dependent-issue FMAs per thread and 64-wide chunk made every K = 500 tile
// a ~12 us chain; with 128 threads the per-chunk FMA chain halves and twice the warps hide the chunk's global round trip.)
constexpr int kTileThreads = 128;

template <int GATHER, typename Sync>
__device__ __forceinline__ void gemm_tile(const GemmJob& J, int m0, int n0, bool first_m_tile, int tid,
                                          float (*As)[TK][TS + 4], float (*Bs)[TK][TS + 4], Sync sync) {
    const int tx = tid & 7, ty = tid >> 3;      // 8 x 16 threads, 2 rows x 4 columns each
    float acc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float csum = 0.f;                            // column-sum lane (threads 0..31 own column n0+tid)
    const bool do_colsum = J.colsum != nullptr && first_m_tile;
    const bool a_ofast = J.a.so <= J.a.sr, b_ofast = J.b.so <= J.b.sr;

    constexpr int EPT = TS * TK / kTileThreads;  // elements per thread per operand and chunk
    float ra[EPT], rb[EPT];
    auto fetch_chunk = [&](int r0) {
        // TS*TK elements per operand; the faster-varying thread index follows the contiguous memory direction
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int f = tid + e * kTileThreads;
            int o, r;
            if (a_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            ra[e] = (m0 + o < J.M && r0 + r < J.R) ? __ldcg(J.a.p + a_offset<GATHER>(J.a, m0 + o, r0 + r)) : 0.f;
            if (b_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            rb[e] = (n0 + o < J.N && r0 + r < J.R) ? __ldcg(J.b.p + (long long)(n0 + o) * J.b.so + (long long)(r0 + r) * J.b.sr) : 0.f;
        }
    };
    fetch_chunk(0);
    int buf = 0;
    for (int r0 = 0; r0 < J.R; r0 += TK, buf ^= 1) {
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int f = tid + e * kTileThreads;
            int o, r;
            if (a_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            As[buf][r][o] = ra[e];
            if (b_ofast) { o = f & 31; r = f >> 5; } else { r = f & (TK - 1); o = f / TK; }
            Bs[buf][r][o] = rb[e];
        }
        sync();
        if (r0 + TK < J.R) fetch_chunk(r0 + TK);
#pragma unroll
        for (int k = 0; k < TK; ++k) {
            const float2 a = *reinterpret_cast<const float2*>(&As[buf][k][ty * 2]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float av[2] = {a.x, a.y};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (do_colsum && tid < 32) {
#pragma unroll
            for (int k = 0; k < TK; ++k) csum += Bs[buf][k][tid];
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int m = m0 + ty * 2 + i;
        if (m >= J.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= J.N) continue;
            float v = acc[i][j] + (J.bias ? __ldcg(J.bias + n) : 0.f);
            if (J.relu) v = fmaxf(v, 0.f);
            if (J.mask) v = __ldcg(J.mask + (long long)m * J.ldc + n) > 0.f ? v : 0.f;
            J.c[(long long)m * J.ldc + n] = v;
        }
    }
    if (do_colsum && tid < 32 && n0 + tid < J.N) J.colsum[n0 + tid] = csum;
    sync();          // the next tile of this group reuses As / Bs
}

template <int GATHER>
__global__ void __launch_bounds__(kTileThreads)
small_gemm_kernel(const __grid_constant__ GemmBatch batch) {
    const GemmJob& J = batch.job[blockIdx.z];
    const int m0 = blockIdx.x * TS, n0 = blockIdx.y * TS;
    if (m0 >= J.M || n0 >= J.N) return;
    // double-buffered tiles: the global loads of chunk i+1 are in flight (in registers) while chunk i is multiplied
    __shared__ __align__(16) float As[2][TK][TS + 4];
    __shared__ __align__(16) float Bs[2][TK][TS + 4];
    gemm_tile<GATHER>(J, m0, n0, blockIdx.x == 0, threadIdx.x, As, Bs, [] { __syncthreads(); });
}

int32_t launch_small_gemm(const GemmBatch& b, int njobs, cudaStream_t s) {
    int maxM = 0, maxN = 0;
    for (int i = 0; i < njobs; ++i) {
        if (b.job[i].M > maxM) maxM = b.job[i].M;
        if (b.job[i].N > maxN) maxN = b.job[i].N;
    }
    if (maxM == 0 || maxN == 0) return CPB_OK;
    dim3 grid(cdiv(maxM, TS), cdiv(maxN, TS), njobs);
    const int gather = b.job[0].a.gather == nullptr ? 0 : (b.job[0].a.gather_on_o ? 1 : 2);   // same for all jobs of a batch
    if (gather == 0) small_gemm_kernel<0><<<grid, kTileThreads, 0, s>>>(b);
    else if (gather == 1) small_gemm_kernel<1><<<grid, kTileThreads, 0, s>>>(b);
    else small_gemm_kernel<2><<<grid, kTileThreads, 0, s>>>(b);
    CPB_LAUNCHED();
    return CPB_OK;
}

// Y[B,N] = act(X[B,K] W[K,N] + b)
__host__ __device__ GemmJob fwd_job(const float* x, const int32_t* idx, int B, int K, const float* w, int N, const float* bias,
                float* y, int relu) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{x, K, 1, idx, 1};
    j.b = Operand{w, 1, N, nullptr, 0};
    j.M = B; j.N = N; j.R = K; j.c = y; j.ldc = N; j.bias = bias; j.relu = relu;
    return j;
}
// dX[B,K] = (dY[B,N] W[K,N]^T) * (H > 0)
__host__ __device__ GemmJob bwd_data_job(const float* dy, int B, int N, const float* w, int K, const float* h, float* dx) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{dy, N, 1, nullptr, 0};
    j.b = Operand{w, N, 1, nullptr, 0};       // b(k, n) = W[k*N + n]
    j.M = B; j.N = K; j.R = N; j.c = dx; j.ldc = K; j.mask = h;
    return j;
}
// gW[K,N] = X[B,K]^T dY[B,N];  gb[N] = colsum(dY)
__host__ __device__ GemmJob bwd_weight_job(const float* x, const int32_t* idx, int B, int K, const float* dy, int N, float* gw, float* gb) {
    GemmJob j;
    memset(&j, 0, sizeof(j));
    j.a = Operand{x, 1, K, idx, 0};           // a(k, b) = X[b*K + k]
    j.b = Operand{dy, 1, N, nullptr, 0};      // b(n, b) = dY[b*N + n]
    j.M = K; j.N = N; j.R = B; j.c = gw; j.ldc = N; j.colsum = gb;
    return j;
}

// ---------------------------------------------------------------------------------------------
// per-sample head: action mean, value, log-prob, ratio, losses and the gradients w.r.t. the two
// trunk outputs (Hp and Hv wide).  One warp per sample.
// ---------------------------------------------------------------------------------------------
constexpr float kLogSqrt2Pi = 0.9189385175704956f;
constexpr float kEntropyConst = 1.4189385175704956f;
constexpr int kMaxActions = 4;
constexpr int kMaxPersistentCtas = 1024;   // upper bound of the persistent learn() grid (one CTA per SM)

struct HeadArgs {
    const float* hp;       // [B,Hp] policy trunk output (post-relu)
    const float* hv;       // [B,Hv] value trunk output (post-relu), may be null (old policy)
    const float* wm; const float* bm; const float* logstd;   // action head
    const float* wv; const float* bv;                        // value head
    const float* actions; const float* returns; const float* adv;   // [T,A], [T], [T] (gathered through idx)
    const int32_t* idx;
    const float* logp_old_in;   // [T] gathered through idx (learn path) or [B] ungathered (train_step path)
    int logp_old_gathered;
    int B, Hp, Hv, A;
    float low[kMaxActions], high[kMaxActions];
    float eps_clip, value_scale, entropy_scale;
    // outputs
    float* logp_out;       // [B] (old-policy pass: log-prob only)
    float* mu_out;         // [B,A] or null
    float* v_out;          // [B] or null
    float* dpre;           // [B,A] gradient w.r.t. the action head pre-activation
    float* dv;             // [B]   gradient w.r.t. the value output
    float* dhp;            // [B,Hp] masked gradient w.r.t. policy trunk output
    float* dhv;            // [B,Hv] masked gradient w.r.t. value trunk output
    float* partial;        // [nblocks][8]: policy, value, ratio sums, logstd grads (3..3+A), approx-KL sum (7)
    const float* noise;    // predict path: [B,A] or null
    float* action_out;     // predict path
    int kl_term;           // training head: add (r - 1) - log r to slot 7 (options entry points only)
    // categorical head only (A = K components): N logits, component k at [coff[k], coff[k+1]); dpre / mu_out are [B,N]
    int N;
    int coff[kMaxActions + 1];
};

// mode 0: log-prob only (old policy); mode 1: full training head; mode 2: predict (mu / sampled action, value)
// one sample (row b) by one warp; MODE 1 adds its loss terms to vals[8]
template <int MODE>
__device__ __forceinline__ void gauss_head_row(const HeadArgs& a, int b, int lane, float* vals) {
    {
        const float* h = a.hp + (long long)b * a.Hp;
        const float* g = MODE != 0 ? a.hv + (long long)b * a.Hv : nullptr;
        float pre[kMaxActions] = {0.f, 0.f, 0.f, 0.f};
        float vsum = 0.f;
        // one loop over both trunk outputs: with Hp == Hv every lane sums in the order of a fused loop
        const int hmax = MODE != 0 && a.Hv > a.Hp ? a.Hv : a.Hp;
        for (int j = lane; j < hmax; j += 32) {
            if (j < a.Hp) {
                const float hv = h[j];
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k)
                    if (k < a.A) pre[k] = fmaf(hv, a.wm[j * a.A + k], pre[k]);
            }
            if (MODE != 0 && j < a.Hv) vsum = fmaf(g[j], a.wv[j], vsum);
        }
#pragma unroll
        for (int k = 0; k < kMaxActions; ++k) pre[k] = warp_sum(pre[k]);
        if (MODE != 0) vsum = warp_sum(vsum);
        const int row = a.idx != nullptr ? a.idx[b] : b;
        float t[kMaxActions], mu[kMaxActions], diff[kMaxActions], sigma[kMaxActions];
        float logp = 0.f;
#pragma unroll
        for (int k = 0; k < kMaxActions; ++k) {
            if (k >= a.A) continue;
            t[k] = tanhf(pre[k] + a.bm[k]);
            mu[k] = a.low[k] + ((t[k] + 1.f) * 0.5f) * (a.high[k] - a.low[k]);
            sigma[k] = expf(a.logstd[k]);
            if (MODE != 2) {
                diff[k] = (a.actions[(long long)row * a.A + k] - mu[k]) / sigma[k];
                logp += -0.5f * diff[k] * diff[k] - (kLogSqrt2Pi + a.logstd[k]);
            }
        }
        if (MODE == 0) {
            if (lane == 0) a.logp_out[b] = logp;
        } else if (MODE == 2) {
            const float v = vsum + a.bv[0];
            if (lane == 0) {
                a.v_out[b] = v;
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k) {
                    if (k >= a.A) continue;
                    float act = mu[k];
                    if (a.noise != nullptr) act = fminf(fmaxf(fmaf(a.noise[(long long)b * a.A + k], sigma[k], mu[k]), a.low[k]), a.high[k]);
                    a.action_out[(long long)b * a.A + k] = act;
                }
            }
        } else {
            const float v = vsum + a.bv[0];
            const float logp_old = a.logp_old_in[a.logp_old_gathered ? row : b];
            const float ratio = expf(logp - logp_old);
            const float adv = a.adv[row], ret = a.returns[row];
            const float unclipped = ratio * adv;
            const float clipped = fminf(fmaxf(ratio, 1.f - a.eps_clip), 1.f + a.eps_clip) * adv;
            const float inv_b = 1.f / (float)a.B;
            // d(-mean(min(u, c)))/d ratio: tf.minimum routes to u when u <= c; the clipped branch has
            // zero slope outside the clip range (inside it u == c and the first branch is taken).
            const float dratio = unclipped <= clipped ? -adv * inv_b : 0.f;
            const float dlogp = dratio * ratio;
            const float dvv = a.value_scale * 2.f * inv_b * (v - ret);
            float dp[kMaxActions] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < kMaxActions; ++k) {
                if (k >= a.A) continue;
                const float dmu = dlogp * diff[k] / sigma[k];
                dp[k] = dmu * 0.5f * (a.high[k] - a.low[k]) * (1.f - t[k] * t[k]);
            }
            if (lane == 0) {
                a.dv[b] = dvv;
#pragma unroll
                for (int k = 0; k < kMaxActions; ++k)
                    if (k < a.A) a.dpre[(long long)b * a.A + k] = dp[k];
                if (a.mu_out != nullptr)
#pragma unroll
                    for (int k = 0; k < kMaxActions; ++k)
                        if (k < a.A) a.mu_out[(long long)b * a.A + k] = mu[k];
                if (a.v_out != nullptr) a.v_out[b] = v;
            }
            for (int j = lane; j < hmax; j += 32) {
                if (j < a.Hp) {
                    float s = 0.f;
#pragma unroll
                    for (int k = 0; k < kMaxActions; ++k)
                        if (k < a.A) s = fmaf(dp[k], a.wm[j * a.A + k], s);
                    a.dhp[(long long)b * a.Hp + j] = h[j] > 0.f ? s : 0.f;
                }
                if (j < a.Hv) a.dhv[(long long)b * a.Hv + j] = g[j] > 0.f ? dvv * a.wv[j] : 0.f;
            }
            vals[0] += fminf(unclipped, clipped);
            vals[1] += (v - ret) * (v - ret);
            vals[2] += ratio;
#pragma unroll
            for (int k = 0; k < kMaxActions; ++k)
                if (k < a.A) vals[3 + k] += dlogp * (diff[k] * diff[k] - 1.f);
            if (a.kl_term) vals[7] += (ratio - 1.f) - (logp - logp_old);   // approximate KL (Stable-Baselines3's estimator)
        }
    }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// logit i (< 64) of a row whose lane l holds logits l in v0 and l + 32 in v1; i is the same in every lane
__device__ __forceinline__ float logit_at(float v0, float v1, int i) { return __shfl_sync(0xffffffffu, i < 32 ? v0 : v1, i & 31); }

// The categorical head of row b (one warp): logits z = h_P W + b with lane l owning logits l and l + 32, one softmax per
// component (segmented warp reductions over a.coff), log-prob of the taken indices, entropy, and in MODE 1 the gradient
//   dz_ki = dlogp (1[i = a_k] - p_ki) + (entropy_scale / B) p_ki (log p_ki + H_k)
// into dpre [B,N] and the masked dh_P.  Every sum has a fixed order, so a repeated call is bit-identical.
template <int MODE>
__device__ __forceinline__ void cat_head_row(const HeadArgs& a, int b, int lane, float* vals) {
    const float* h = a.hp + (long long)b * a.Hp;
    const int N = a.N, K = a.A;
    const bool has0 = lane < N, has1 = lane + 32 < N;
    // logits: the rows of W are read coalesced, h 32 values at a time and broadcast lane to lane
    float z0 = 0.f, z1 = 0.f;
    for (int j0 = 0; j0 < a.Hp; j0 += 32) {
        const float hl = j0 + lane < a.Hp ? h[j0 + lane] : 0.f;
        const int n = a.Hp - j0 < 32 ? a.Hp - j0 : 32;
        for (int t = 0; t < n; ++t) {
            const float hj = __shfl_sync(0xffffffffu, hl, t);
            const float* w = a.wm + (long long)(j0 + t) * N;
            if (has0) z0 = fmaf(hj, w[lane], z0);
            if (has1) z1 = fmaf(hj, w[lane + 32], z1);
        }
    }
    if (has0) z0 += a.bm[lane];
    if (has1) z1 += a.bm[lane + 32];
    // component of each owned logit, and the per-component softmax: max, sum of exp, entropy (warp-uniform values)
    int c0 = 0, c1 = 0;
#pragma unroll
    for (int k = 1; k < kMaxActions; ++k)
        if (k < K) { c0 += lane >= a.coff[k]; c1 += lane + 32 >= a.coff[k]; }
    float mx[kMaxActions], lse[kMaxActions], ent[kMaxActions];
    float m0 = 0.f, m1 = 0.f, l0 = 0.f, l1 = 0.f, s0 = 1.f, s1 = 1.f, H0 = 0.f, H1 = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        float v = -INFINITY;
        if (has0 && c0 == k) v = z0;
        if (has1 && c1 == k) v = fmaxf(v, z1);
        mx[k] = warp_max(v);
        if (c0 == k) m0 = mx[k];
        if (c1 == k) m1 = mx[k];
    }
    const float e0 = has0 ? expf(z0 - m0) : 0.f, e1 = has1 ? expf(z1 - m1) : 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        const float s = warp_sum((c0 == k ? e0 : 0.f) + (c1 == k ? e1 : 0.f));
        lse[k] = logf(s);
        if (c0 == k) { l0 = lse[k]; s0 = s; }
        if (c1 == k) { l1 = lse[k]; s1 = s; }
    }
    const float lp0 = has0 ? z0 - m0 - l0 : 0.f, lp1 = has1 ? z1 - m1 - l1 : 0.f;   // log p
    const float p0 = e0 / s0, p1 = e1 / s1;
    float entropy = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        ent[k] = -warp_sum((c0 == k ? p0 * lp0 : 0.f) + (c1 == k ? p1 * lp1 : 0.f));
        entropy += ent[k];
        if (c0 == k) H0 = ent[k];
        if (c1 == k) H1 = ent[k];
    }
    (void)mx; (void)lse;
    if (MODE == 2) {
        float vsum = 0.f;
        const float* g = a.hv + (long long)b * a.Hv;
        for (int j = lane; j < a.Hv; j += 32) vsum = fmaf(g[j], a.wv[j], vsum);
        vsum = warp_sum(vsum);
        // greedy: the first largest logit; sampled: the first i with u < cumsum_i p (fp32, index order), else the last
        // index with p > 0.  Every lane runs the same scan on broadcast values; lane 0 writes.
        for (int k = 0; k < K; ++k) {
            const int lo = a.coff[k], hi = a.coff[k + 1];
            int pick = -1, last_pos = 0;
            if (a.noise == nullptr) {
                float best = -INFINITY;
                pick = 0;
                for (int i = lo; i < hi; ++i) {
                    const float zi = logit_at(z0, z1, i);
                    if (zi > best) { best = zi; pick = i - lo; }
                }
            } else {
                const float u = a.noise[(long long)b * K + k];
                float c = 0.f;
                for (int i = lo; i < hi; ++i) {
                    const float pi = logit_at(p0, p1, i);
                    c += pi;
                    if (pick < 0 && u < c) pick = i - lo;
                    if (pi > 0.f) last_pos = i - lo;
                }
                if (pick < 0) pick = last_pos;
            }
            if (lane == 0) a.action_out[(long long)b * K + k] = (float)pick;
        }
        if (lane == 0) a.v_out[b] = vsum + a.bv[0];
        return;
    }
    // log-prob of the taken indices (clamped into each component's range)
    const int row = a.idx != nullptr ? a.idx[b] : b;
    float logp = 0.f;
    int t0 = -1, t1 = -1;   // the taken index of the component of logit lane / lane + 32
#pragma unroll
    for (int k = 0; k < kMaxActions; ++k) {
        if (k >= K) continue;
        const float av = a.actions[(long long)row * K + k];
        const int t = a.coff[k] + (int)fminf(fmaxf(av, 0.f), (float)(a.coff[k + 1] - a.coff[k] - 1));
        logp += logit_at(lp0, lp1, t);
        if (c0 == k) t0 = t;
        if (c1 == k) t1 = t;
    }
    if (MODE == 0) {
        if (lane == 0) a.logp_out[b] = logp;
        return;
    }
    const float* g = a.hv + (long long)b * a.Hv;
    float vsum = 0.f;
    for (int j = lane; j < a.Hv; j += 32) vsum = fmaf(g[j], a.wv[j], vsum);
    vsum = warp_sum(vsum);
    const float v = vsum + a.bv[0];
    const float logp_old = a.logp_old_in[a.logp_old_gathered ? row : b];
    const float ratio = expf(logp - logp_old);
    const float adv = a.adv[row], ret = a.returns[row];
    const float unclipped = ratio * adv;
    const float clipped = fminf(fmaxf(ratio, 1.f - a.eps_clip), 1.f + a.eps_clip) * adv;
    const float inv_b = 1.f / (float)a.B;
    const float dratio = unclipped <= clipped ? -adv * inv_b : 0.f;   // the Gaussian head's tf.minimum rule
    const float dlogp = dratio * ratio;
    const float dvv = a.value_scale * 2.f * inv_b * (v - ret);
    const float es = a.entropy_scale * inv_b;
    const float dz0 = has0 ? dlogp * ((lane == t0 ? 1.f : 0.f) - p0) + es * p0 * (lp0 + H0) : 0.f;
    const float dz1 = has1 ? dlogp * ((lane + 32 == t1 ? 1.f : 0.f) - p1) + es * p1 * (lp1 + H1) : 0.f;
    if (has0) a.dpre[(long long)b * N + lane] = dz0;
    if (has1) a.dpre[(long long)b * N + lane + 32] = dz1;
    if (lane == 0) {
        a.dv[b] = dvv;
        if (a.v_out != nullptr) a.v_out[b] = v;
    }
    // dh_P[j] = sum_i dz_i W[j, i] (i in index order), masked by h_P > 0; lane l owns j = j0 + l
    for (int j0 = 0; j0 < a.Hp; j0 += 32) {
        const int j = j0 + lane;
        const float* w = a.wm + (long long)(j < a.Hp ? j : 0) * N;
        float s = 0.f;
        for (int i = 0; i < N; ++i) s = fmaf(logit_at(dz0, dz1, i), w[i], s);
        if (j < a.Hp) a.dhp[(long long)b * a.Hp + j] = h[j] > 0.f ? s : 0.f;
    }
    for (int j = lane; j < a.Hv; j += 32) a.dhv[(long long)b * a.Hv + j] = g[j] > 0.f ? dvv * a.wv[j] : 0.f;
    vals[0] += fminf(unclipped, clipped);
    vals[1] += (v - ret) * (v - ret);
    vals[2] += ratio;
    vals[3] += entropy;
    if (a.kl_term) vals[7] += (ratio - 1.f) - (logp - logp_old);
}

// CAT: 0 = the Gaussian head, 1 = the categorical head
template <int MODE, int CAT>
__device__ __forceinline__ void head_row(const HeadArgs& a, int b, int lane, float* vals) {
    if constexpr (CAT != 0) cat_head_row<MODE>(a, b, lane, vals);
    else gauss_head_row<MODE>(a, b, lane, vals);
}

// CTA-level sum of the 8 warps' loss terms -> partial[block][8] (fixed order: deterministic)
__device__ __forceinline__ void head_block_reduce(const float* vals, float (*red)[8], float* partial_out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < 8; ++k) red[warp][k] = vals[k];
    __syncthreads();
    if (threadIdx.x < 8) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
        partial_out[threadIdx.x] = s;
    }
    __syncthreads();
}

template <int MODE, int CAT>
__global__ void __launch_bounds__(256)
ppo_head_kernel(const __grid_constant__ HeadArgs a) {
    __shared__ float red[8][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    float vals[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (b < a.B) head_row<MODE, CAT>(a, b, lane, vals);
    if (MODE == 1) head_block_reduce(vals, red, a.partial + blockIdx.x * 8);
}

template <int MODE>
void launch_head(const HeadShape& hs, int B, const HeadArgs& h, cudaStream_t s) {
    if (hs.cat) ppo_head_kernel<MODE, 1><<<cdiv(B, 8), 256, 0, s>>>(h);
    else ppo_head_kernel<MODE, 0><<<cdiv(B, 8), 256, 0, s>>>(h);
}

// The per-call guards of the cpb_ppo_*_opts entry points (cpb_ppo_learn_options).  stop == nullptr on every other entry
// point: then none of the guard code runs and the metrics rows are 5 wide.
//   stop: device word, 0 while the update runs.  ppo_finalize sets it to 1 at the minibatch whose approx_kl exceeds
//         kl_limit and to 2 at every minibatch evaluated after that; Adam skips every step while it is non-zero.
//   clip: device float[1], the current minibatch's gradient scale min(1, max_norm / (norm + 1e-6)) (1 when max_norm == 0).
struct Guards {
    uint32_t* stop;
    float* clip;
    float* norm_partial;   // [kMaxPersistentCtas] per-block sums of squares of the gradient
    uint32_t* counter;     // blocks of grad_norm_kernel done (back to 0 when it ends)
    int32_t* steps;        // Adam steps applied (nullable)
    float max_norm;        // 0: no clipping
    float kl_limit;        // 1.5 * target_kl; 0: no stop
};

// metrics[5] = policy_loss, value_loss, entropy_loss, loss, mean ratio; grads[logstd], value-bias etc.
// With guards, metrics rows are 7 wide: [5] = approx_kl (written here), [6] = the pre-clip gradient norm (written by the
// norm reduction); a minibatch evaluated after the stop gets a NaN row.
// CAT: the categorical head's entropy is the batch mean of slot 3 (sum_b H_b), and there is no logstd gradient.
template <int CAT>
__device__ __forceinline__ void ppo_finalize(const float* partial, int nblocks, int B, int A, const float* logstd, float value_scale,
                                             float entropy_scale, float* glogstd, float* metrics, float* tot /* shared [8] */,
                                             const Guards& g) {
    if (threadIdx.x < 8) {
        float s = 0.f;
        for (int i = 0; i < nblocks; ++i) s += __ldcg(partial + i * 8 + threadIdx.x);
        tot[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float inv_b = 1.f / (float)B;
        float ent = 0.f;
        if constexpr (CAT != 0) ent = tot[3] * inv_b;
        else
            for (int k = 0; k < A; ++k) {
                ent += kEntropyConst + logstd[k];
                glogstd[k] = tot[3 + k] - entropy_scale;
            }
        const float pl = tot[0] * inv_b;
        const float vl = tot[1] * inv_b * value_scale;
        const float el = ent * entropy_scale;
        if (g.stop != nullptr && __ldcg(g.stop) != 0u) {
            *g.stop = 2u;
            if (metrics != nullptr)
                for (int k = 0; k < 7; ++k) metrics[k] = __int_as_float(0x7fc00000);
        } else {
            if (metrics != nullptr) {
                metrics[0] = pl; metrics[1] = vl; metrics[2] = el; metrics[3] = -pl + vl - el; metrics[4] = tot[2] * inv_b;
            }
            if (g.stop != nullptr) {
                const float kl = tot[7] * inv_b;
                if (metrics != nullptr) metrics[5] = kl;
                if (g.kl_limit > 0.f && kl > g.kl_limit) *g.stop = 1u;
            }
        }
    }
    __syncthreads();
}

template <int CAT>
__global__ void ppo_finalize_kernel(const float* __restrict__ partial, int nblocks, int B, int A,
                                    const float* __restrict__ logstd, float value_scale, float entropy_scale,
                                    float* __restrict__ glogstd, float* __restrict__ metrics, const Guards g) {
    __shared__ float tot[8];
    ppo_finalize<CAT>(partial, nblocks, B, A, logstd, value_scale, entropy_scale, glogstd, metrics, tot, g);
}

// ---------------------------------------------------------------------------------------------
// global L2 norm of the gradient (torch.nn.utils.clip_grad_norm_ over the 13 policy/ tensors; the layout's zero padding
// adds nothing).  Every sum has a fixed order, so a repeated call is bit-identical.
// ---------------------------------------------------------------------------------------------
constexpr int kNormBlocks = 256, kNormThreads = 256;

// sum of v over the CTA's threads in a fixed order, returned to every thread; red: shared [blockDim.x / 32]
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    __syncthreads();                  // red may still be read by a previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

// this thread's share of sum(g^2): float4 elements k = first, first + stride, ...
__device__ __forceinline__ float sumsq_share(const float4* g, long long n4, long long first, long long stride) {
    float s = 0.f;
    for (long long k = first; k < n4; k += stride) {
        const float4 v = __ldcg(g + k);
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    }
    return s;
}

__device__ __forceinline__ float clip_coefficient(float sumsq, float max_norm) {
    if (max_norm <= 0.f) return 1.f;
    const float c = max_norm / (sqrtf(sumsq) + 1e-6f);
    return c < 1.f ? c : 1.f;
}

// partial sums per block, then the last block to finish sums the partials in block order: clip coefficient, metrics[6]
__global__ void __launch_bounds__(kNormThreads)
grad_norm_kernel(const float4* __restrict__ g, long long n4, const Guards gd, float* __restrict__ metrics) {
    __shared__ float red[kNormThreads / 32];
    __shared__ bool last;
    const float s = block_sum(sumsq_share(g, n4, (long long)blockIdx.x * blockDim.x + threadIdx.x, (long long)gridDim.x * blockDim.x), red);
    if (threadIdx.x == 0) {
        gd.norm_partial[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(gd.counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    float t = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(gd.norm_partial + i);
    t = block_sum(t, red);
    if (threadIdx.x == 0) {
        gd.clip[0] = clip_coefficient(t, gd.max_norm);
        if (metrics != nullptr && __ldcg(gd.stop) != 2u) metrics[6] = sqrtf(t);
        *gd.counter = 0u;
    }
}

int32_t launch_grad_norm(const float* grads, long long n, const Guards& gd, float* metrics, cudaStream_t s) {
    grad_norm_kernel<<<kNormBlocks, kNormThreads, 0, s>>>(reinterpret_cast<const float4*>(grads), n / 4, gd, metrics);
    CPB_LAUNCHED();
    return CPB_OK;
}

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

int32_t launch_gae_segments(const double* rewards, const double* values, const double* bootstrap, const double* dones,
                            const int32_t* offsets, int num_segments, int rows, double gamma, double lam, double* adv,
                            double* ret_out, double* advn_out, float* ret32, float* advn32, cudaStream_t s) {
    gae_segments_scan_kernel<<<num_segments, kGaeThreads, 0, s>>>(rewards, values, bootstrap, dones, offsets, gamma, lam, adv);
    CPB_LAUNCHED();
    gae_normalise_kernel<<<1, kGaeThreads, 0, s>>>(adv, values, rows, ret_out, advn_out, ret32, advn32);
    CPB_LAUNCHED();
    return CPB_OK;
}

// ---------------------------------------------------------------------------------------------
// workspace plan
// ---------------------------------------------------------------------------------------------
struct PpoPlan {
    float* h[kMaxPpoDepth];    // layer l of both trunks: [B,Wp_l] policy then [B,Wv_l] value (a trunk past its depth: none)
    float* dh[kMaxPpoDepth];   // same shapes: masked gradients w.r.t. the layer outputs
    float* oh[kMaxPpoDepth];   // old-policy trunk [rows,Wp_l], l < P
    float *logp_old;       // [rows]
    float *dpre, *dv, *partial;
    float *ret32, *adv32;  // [T]
    double* gae_scratch;   // [T]
    float* norm_partial;   // [kMaxPersistentCtas]  guards of the options entry points (Guards)
    uint32_t* guard_words; // [4]: stop, counter, clip (as float bits), unused
    int64_t bytes;
    bool ok;
};

// width of trunk t's layer l, 0 past its depth
__host__ __device__ __forceinline__ int width_or_0(const cpb_ppo_spec& sp, int t, int l) {
    return l < trunk_depth(sp, t) ? trunk_width(sp, t, l) : 0;
}
// trunk t's part of a per-layer buffer (pl.h[l] / pl.dh[l]) at batch B
__host__ __device__ __forceinline__ float* trunk_buf(float* const* bufs, const cpb_ppo_spec& sp, int t, int l, int B) {
    return bufs[l] + (t ? (long long)B * width_or_0(sp, 0, l) : 0);
}

PpoPlan make_ppo_plan(void* ws, int64_t ws_bytes, const cpb_ppo_spec* sp, const HeadShape& hs, int max_batch, int horizon) {
    PpoPlan p;
    memset(&p, 0, sizeof(p));
    Arena a(ws, ws_bytes);
    const int64_t B = max_batch;
    const int64_t rows = horizon > max_batch ? horizon : max_batch;
    const int D = max_depth(*sp);
    for (int l = 0; l < D; ++l) p.h[l] = a.take<float>(B * (width_or_0(*sp, 0, l) + width_or_0(*sp, 1, l)));
    for (int l = D - 1; l >= 0; --l) p.dh[l] = a.take<float>(B * (width_or_0(*sp, 0, l) + width_or_0(*sp, 1, l)));
    for (int l = 0; l < sp->num_policy; ++l) p.oh[l] = a.take<float>(rows * sp->policy_sizes[l]);
    p.logp_old = a.take<float>(rows);
    p.dpre = a.take<float>(B * (hs.cat ? hs.N : kMaxActions));
    p.dv = a.take<float>(B);
    p.partial = a.take<float>((int64_t)(cdiv(B, 8) > kMaxPersistentCtas ? cdiv(B, 8) : kMaxPersistentCtas) * 8);
    p.ret32 = a.take<float>(rows);
    p.adv32 = a.take<float>(rows);
    p.gae_scratch = a.take<double>(rows);
    p.norm_partial = a.take<float>(kMaxPersistentCtas);
    p.guard_words = a.take<uint32_t>(4);
    p.bytes = a.off;
    p.ok = ws == nullptr || !a.overflow;
    return p;
}

int32_t check_ppo_spec(const cpb_ppo_spec* sp) {
    CPB_REQUIRE(sp != nullptr, "ppo spec is NULL");
    const cpb_ppo_config* c = &sp->base;
    CPB_REQUIRE(c->hidden1 == 0 && c->hidden2 == 0,
                "ppo spec: base.hidden1 / base.hidden2 must be 0 (the widths are policy_sizes / value_sizes), got %d, %d",
                c->hidden1, c->hidden2);
    CPB_REQUIRE(c->state_dim >= 1, "ppo: state_dim must be >= 1, got %d", c->state_dim);
    CPB_REQUIRE(c->num_actions >= 1 && c->num_actions <= kMaxActions, "ppo: num_actions must be in [1,%d]", kMaxActions);
    CPB_REQUIRE(sp->num_policy >= 1 && sp->num_policy <= kMaxPpoDepth && sp->num_value >= 1 && sp->num_value <= kMaxPpoDepth,
                "ppo spec: each trunk needs 1 to %d hidden layers, got %d (policy) and %d (value)", kMaxPpoDepth,
                sp->num_policy, sp->num_value);
    for (int t = 0; t < 2; ++t)
        for (int l = 0; l < trunk_depth(*sp, t); ++l)
            CPB_REQUIRE(trunk_width(*sp, t, l) >= 1, "ppo spec: %s layer %d has width %d (must be >= 1)",
                        t ? "value" : "policy", l, trunk_width(*sp, t, l));
    return CPB_OK;
}

// A cpb_ppo_cat_spec -> its HeadShape, refusing a bad one (the Gaussian spec's checks first)
int32_t cat_head(const cpb_ppo_cat_spec* cs, HeadShape* hs) {
    CPB_REQUIRE(cs != nullptr, "ppo categorical spec is NULL");
    CPB_TRY(check_ppo_spec(&cs->spec));
    const cpb_ppo_config& c = cs->spec.base;
    for (int k = 0; k < kMaxActions; ++k)
        CPB_REQUIRE(c.action_low[k] == 0.f && c.action_high[k] == 0.f,
                    "ppo categorical spec: spec.base.action_low / action_high must be 0 (component %d)", k);
    memset(hs, 0, sizeof(*hs));
    hs->cat = 1;
    hs->K = c.num_actions;
    for (int k = 0; k < hs->K; ++k) {
        const int n = cs->num_categories[k];
        CPB_REQUIRE(n >= 2 && n <= kMaxLogits, "ppo categorical spec: component %d has %d categories (must be 2..%d)", k, n,
                    kMaxLogits);
        hs->off[k + 1] = hs->off[k] + n;
    }
    hs->N = hs->off[hs->K];
    for (int k = hs->K + 1; k < 5; ++k) hs->off[k] = hs->N;
    CPB_REQUIRE(hs->N <= kMaxLogits, "ppo categorical spec: %d logits in all (at most %d)", hs->N, kMaxLogits);
    return CPB_OK;
}

HeadArgs head_args(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const float* params, int B) {
    const cpb_ppo_config* c = &sp->base;
    HeadArgs h;
    memset(&h, 0, sizeof(h));
    h.wm = params + L.off[L.wm()]; h.bm = params + L.off[L.bm()]; h.logstd = params + L.off[L.logstd()];
    h.wv = params + L.off[L.wv()]; h.bv = params + L.off[L.bv()];
    h.B = B; h.Hp = trunk_last(*sp, 0); h.Hv = trunk_last(*sp, 1); h.A = c->num_actions;
    for (int k = 0; k < kMaxActions; ++k) { h.low[k] = c->action_low[k]; h.high[k] = c->action_high[k]; }
    h.eps_clip = c->epsilon; h.value_scale = c->value_scale; h.entropy_scale = c->entropy_scale;
    h.N = hs.N;
    for (int k = 0; k < 5; ++k) h.coff[k] = hs.off[k];
    return h;
}

// log pi_old(a|s) for `rows` samples (optionally gathered)
int32_t run_old_logp(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, const float* params_old,
                     const float* states, const float* actions, const int32_t* idx, int rows, cudaStream_t s) {
    GemmBatch gb;
    for (int l = 0; l < sp->num_policy; ++l) {
        gb.job[0] = fwd_job(l ? pl.oh[l - 1] : states, l ? nullptr : idx, rows, trunk_in(*sp, 0, l),
                            params_old + L.off[L.w(0, l)], sp->policy_sizes[l], params_old + L.off[L.b(0, l)], pl.oh[l], 1);
        CPB_TRY(launch_small_gemm(gb, 1, s));
    }
    HeadArgs h = head_args(sp, hs, L, params_old, rows);
    h.hp = pl.oh[sp->num_policy - 1]; h.actions = actions; h.idx = idx; h.logp_out = pl.logp_old;
    launch_head<0>(hs, rows, h, s);
    CPB_LAUNCHED();
    return CPB_OK;
}

// Forward jobs of layer l: one per trunk that has it (layer 0 reads the states through idx)
__host__ __device__ __forceinline__ int trunk_fwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       const float* params, const float* states, const int32_t* idx, int B,
                                                       int l, GemmJob* jobs) {
    int n = 0;
    for (int t = 0; t < 2; ++t) {
        if (l >= trunk_depth(sp, t)) continue;
        const float* in = l ? trunk_buf(pl.h, sp, t, l - 1, B) : states;
        jobs[n++] = fwd_job(in, l ? nullptr : idx, B, trunk_in(sp, t, l), params + L.off[L.w(t, l)], trunk_width(sp, t, l),
                            params + L.off[L.b(t, l)], trunk_buf(pl.h, sp, t, l, B), 1);
    }
    return n;
}

// Backward jobs of layer l: per trunk that has it, the weight and bias gradients and (l > 0) the masked data gradient into
// layer l - 1.  Layer 0 reads the states through idx, so its jobs gather (GATHER 2 when idx != null) and the rest do not.
__host__ __device__ __forceinline__ int trunk_bwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       const float* params, float* grads, const float* states,
                                                       const int32_t* idx, int B, int l, GemmJob* jobs) {
    int n = 0;
    for (int t = 0; t < 2; ++t) {
        if (l >= trunk_depth(sp, t)) continue;
        const float* in = l ? trunk_buf(pl.h, sp, t, l - 1, B) : states;
        jobs[n++] = bwd_weight_job(in, l ? nullptr : idx, B, trunk_in(sp, t, l), trunk_buf(pl.dh, sp, t, l, B),
                                   trunk_width(sp, t, l), grads + L.off[L.w(t, l)], grads + L.off[L.b(t, l)]);
    }
    if (l > 0)
        for (int t = 0; t < 2; ++t) {
            if (l >= trunk_depth(sp, t)) continue;
            jobs[n++] = bwd_data_job(trunk_buf(pl.dh, sp, t, l, B), B, trunk_width(sp, t, l), params + L.off[L.w(t, l)],
                                     trunk_in(sp, t, l), trunk_buf(pl.h, sp, t, l - 1, B), trunk_buf(pl.dh, sp, t, l - 1, B));
        }
    return n;
}

// Weight and bias gradients of the action and value heads: gWm[Hp,N] = hp^T dpre, gbm = colsum(dpre); gWv[Hv,1] = hv^T dv
// (N: the head's columns, num_actions for the Gaussian head, the logits for the categorical one)
__host__ __device__ __forceinline__ void head_bwd_jobs(const cpb_ppo_spec& sp, const PpoLayout& L, const PpoPlan& pl,
                                                       float* grads, int B, int N, GemmJob* jobs) {
    jobs[0] = bwd_weight_job(trunk_buf(pl.h, sp, 0, sp.num_policy - 1, B), nullptr, B, trunk_last(sp, 0), pl.dpre,
                             N, grads + L.off[L.wm()], grads + L.off[L.bm()]);
    jobs[1] = bwd_weight_job(trunk_buf(pl.h, sp, 1, sp.num_value - 1, B), nullptr, B, trunk_last(sp, 1), pl.dv, 1,
                             grads + L.off[L.wv()], grads + L.off[L.bv()]);
}

int32_t run_trunks(const cpb_ppo_spec* sp, const PpoLayout& L, const PpoPlan& pl, const float* params,
                   const float* states, const int32_t* idx, int B, cudaStream_t s) {
    GemmBatch gb;
    for (int l = 0; l < max_depth(*sp); ++l)
        CPB_TRY(launch_small_gemm(gb, trunk_fwd_jobs(*sp, L, pl, params, states, idx, B, l, gb.job), s));
    return CPB_OK;
}

// forward + loss + gradients for one minibatch; logp_old given (gathered or not)
int32_t run_loss_grad(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, const float* params,
                      const float* states, const float* actions, const float* returns, const float* adv,
                      const int32_t* idx, int B, const float* logp_old, int logp_old_gathered, float* grads,
                      float* metrics, const Guards& gd, cudaStream_t s) {
    const cpb_ppo_config* c = &sp->base;
    const int P = sp->num_policy, V = sp->num_value, D = max_depth(*sp);
    CPB_TRY(run_trunks(sp, L, pl, params, states, idx, B, s));
    HeadArgs h = head_args(sp, hs, L, params, B);
    h.hp = trunk_buf(pl.h, *sp, 0, P - 1, B); h.hv = trunk_buf(pl.h, *sp, 1, V - 1, B);
    h.actions = actions; h.returns = returns; h.adv = adv; h.idx = idx;
    h.logp_old_in = logp_old; h.logp_old_gathered = logp_old_gathered;
    h.dpre = pl.dpre; h.dv = pl.dv; h.dhp = trunk_buf(pl.dh, *sp, 0, P - 1, B); h.dhv = trunk_buf(pl.dh, *sp, 1, V - 1, B);
    h.partial = pl.partial;
    h.kl_term = gd.stop != nullptr;
    const int nblocks = cdiv(B, 8);
    launch_head<1>(hs, B, h, s);
    CPB_LAUNCHED();
    if (hs.cat)
        ppo_finalize_kernel<1><<<1, 32, 0, s>>>(pl.partial, nblocks, B, c->num_actions, nullptr, c->value_scale,
                                                c->entropy_scale, nullptr, metrics, gd);
    else
        ppo_finalize_kernel<0><<<1, 32, 0, s>>>(pl.partial, nblocks, B, c->num_actions, params + L.off[L.logstd()],
                                                c->value_scale, c->entropy_scale, grads + L.off[L.logstd()], metrics, gd);
    CPB_LAUNCHED();
    // one launch per layer, top down, for both trunks: weight gradients and the data gradient into the layer below.  The
    // head weight gradients only need the head kernel's outputs and join the top layer's launch (at two layers per trunk:
    // 6 independent GEMMs), unless that launch gathers the states (one layer in both trunks).
    GemmBatch gb;
    for (int l = D - 1; l >= 0; --l) {
        int n = trunk_bwd_jobs(*sp, L, pl, params, grads, states, idx, B, l, gb.job);
        if (l == D - 1) {
            if (l == 0 && idx != nullptr) {
                GemmBatch hb;
                head_bwd_jobs(*sp, L, pl, grads, B, hs.N, hb.job);
                CPB_TRY(launch_small_gemm(hb, 2, s));
            } else {
                head_bwd_jobs(*sp, L, pl, grads, B, hs.N, gb.job + n);
                n += 2;
            }
        }
        CPB_TRY(launch_small_gemm(gb, n, s));
    }
    return CPB_OK;
}

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
                HeadArgs h;
                h.hp = trunk_buf(pl.h, sp, 0, sp.num_policy - 1, B); h.hv = trunk_buf(pl.h, sp, 1, sp.num_value - 1, B);
                h.wm = params + L.off[L.wm()]; h.bm = params + L.off[L.bm()]; h.logstd = params + L.off[L.logstd()];
                h.wv = params + L.off[L.wv()]; h.bv = params + L.off[L.bv()];
                h.actions = a.actions; h.returns = pl.ret32; h.adv = pl.adv32; h.idx = idx;
                h.logp_old_in = pl.logp_old; h.logp_old_gathered = 1;
                h.B = B; h.Hp = trunk_last(sp, 0); h.Hv = trunk_last(sp, 1); h.A = A;
                for (int k = 0; k < kMaxActions; ++k) { h.low[k] = c.action_low[k]; h.high[k] = c.action_high[k]; }
                h.eps_clip = c.epsilon; h.value_scale = c.value_scale; h.entropy_scale = c.entropy_scale;
                h.logp_out = nullptr; h.mu_out = nullptr; h.v_out = nullptr;
                h.dpre = pl.dpre; h.dv = pl.dv; h.partial = pl.partial;
                h.dhp = trunk_buf(pl.dh, sp, 0, sp.num_policy - 1, B); h.dhv = trunk_buf(pl.dh, sp, 1, sp.num_value - 1, B);
                h.noise = nullptr; h.action_out = nullptr;
                h.kl_term = gd.stop != nullptr;
                if constexpr (CAT != 0) {
                    h.N = a.hs.N;
                    for (int k = 0; k < 5; ++k) h.coff[k] = a.hs.off[k];
                }
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
            // ---- TF ApplyAdam (the arithmetic of adam_kernel), beta powers advanced after the barrier
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
                    mv.x += (gv.x - mv.x) * omb1; mv.y += (gv.y - mv.y) * omb1; mv.z += (gv.z - mv.z) * omb1; mv.w += (gv.w - mv.w) * omb1;
                    vv.x += (gv.x * gv.x - vv.x) * omb2; vv.y += (gv.y * gv.y - vv.y) * omb2;
                    vv.z += (gv.z * gv.z - vv.z) * omb2; vv.w += (gv.w * gv.w - vv.w) * omb2;
                    pv.x -= (mv.x * alpha) / (sqrtf(vv.x) + epsilon); pv.y -= (mv.y * alpha) / (sqrtf(vv.y) + epsilon);
                    pv.z -= (mv.z * alpha) / (sqrtf(vv.z) + epsilon); pv.w -= (mv.w * alpha) / (sqrtf(vv.w) + epsilon);
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

// Everything of the driver's update block after GAE (train.py:178-207): theta_old <- theta, the old policy's
// log-probabilities, and num_epochs x ceil(T / batch_size) minibatch Adam steps reading pl.ret32 / pl.adv32.
int32_t learn_update(const cpb_ppo_spec* sp, const HeadShape& hs, const PpoLayout& L, const PpoPlan& pl, float* params, float* params_old,
                     float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                     const float* states, const float* actions, int T, int num_epochs, int batch_size,
                     const int32_t* perms, float* metrics, const Guards& gd, cudaStream_t s) {
    const int mcols = gd.stop != nullptr ? 7 : 5;
    // theta_old <- theta (PPO.update_old_policy, ppo.py:275-276)
    CPB_CUDA(cudaMemcpyAsync(params_old, params, L.total * sizeof(float), cudaMemcpyDeviceToDevice, s));
    // log pi_old(a_t|s_t) is constant during the update: evaluate it once for all T samples
    CPB_TRY(run_old_logp(sp, hs, L, pl, params_old, states, actions, nullptr, T, s));
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    const int nmb = cdiv(T, batch_size);
    CPB_TRY(learn_persistent_init());
    if (g_learn_grid > 0 && num_epochs > 0) {
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
        return CPB_OK;
    }
    for (int e = 0; e < num_epochs; ++e)
        for (int i = 0; i < nmb; ++i) {
            const int begin = i * batch_size;
            const int B = begin + batch_size <= T ? batch_size : T - begin;
            const int32_t* idx = perms + (long long)e * T + begin;
            float* mt = metrics ? metrics + ((long long)e * nmb + i) * mcols : nullptr;
            CPB_TRY(run_loss_grad(sp, hs, L, pl, params, states, actions, pl.ret32, pl.adv32, idx, B, pl.logp_old, 1,
                                  grads, mt, gd, s));
            if (gd.stop != nullptr) {
                // the minibatches after a stop are still launched (the host cannot know); Adam skips them on the device
                CPB_TRY(launch_grad_norm(grads, L.total, gd, mt, s));
                CPB_TRY(launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s,
                                    gd.stop, gd.clip, gd.steps));
            } else {
                CPB_TRY(launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s));
            }
        }
    return CPB_OK;
}

// cpb_ppo_learn_options -> Guards on the plan's guard scratch, refusing bad options before anything is enqueued.  stop:
// the caller's stop word (train_step), or null for a zeroed word of the call's own (learn).  steps_applied is zeroed.
int32_t make_guards(const cpb_ppo_learn_options* opts, const PpoPlan& pl, uint32_t* stop, int32_t* steps_applied,
                    cudaStream_t s, Guards* gd) {
    float max_norm = 0.f, target_kl = 0.f;
    if (opts != nullptr) { max_norm = opts->max_grad_norm; target_kl = opts->target_kl; }
    CPB_REQUIRE(std::isfinite(max_norm) && max_norm >= 0.f, "ppo options: max_grad_norm must be finite and >= 0 (0 = off)");
    CPB_REQUIRE(std::isfinite(target_kl) && target_kl >= 0.f, "ppo options: target_kl must be finite and >= 0 (0 = off)");
    memset(gd, 0, sizeof(*gd));
    gd->stop = stop != nullptr ? stop : pl.guard_words;
    gd->counter = pl.guard_words + 1;
    gd->clip = reinterpret_cast<float*>(pl.guard_words + 2);
    gd->norm_partial = pl.norm_partial;
    gd->steps = steps_applied;
    gd->max_norm = max_norm;
    gd->kl_limit = (float)(1.5 * (double)target_kl);
    // the plan's own stop word (used when the caller gives none) and the norm reduction's block counter start at 0
    CPB_CUDA(cudaMemsetAsync(pl.guard_words, 0, 2 * sizeof(uint32_t), s));
    if (steps_applied != nullptr) CPB_CUDA(cudaMemsetAsync(steps_applied, 0, sizeof(int32_t), s));
    return CPB_OK;
}

}  // namespace
}  // namespace cpb

using namespace cpb;

// The cpb_ppo_spec and cpb_ppo_cat_spec entry points share one implementation each, on (spec, head shape) of a checked spec
#define CPB_PPO_PLAN(maxb, horizon)                                                            \
    CPB_REQUIRE(workspace != nullptr, "workspace is NULL");                                    \
    PpoPlan pl = make_ppo_plan(workspace, workspace_bytes, spec, hs, maxb, horizon);           \
    if (!pl.ok) {                                                                              \
        cpb::set_error("ppo workspace too small: need %lld bytes, got %lld", (long long)pl.bytes, \
                       (long long)workspace_bytes);                                            \
        return CPB_ERR_WORKSPACE_TOO_SMALL;                                                    \
    }                                                                                          \
    PpoLayout L = make_ppo_layout(spec, hs);                                                   \
    cudaStream_t s = (cudaStream_t)stream;

static int32_t ppo_layout(const cpb_ppo_spec* spec, const HeadShape& hs, int64_t* offsets, int64_t* sizes, int32_t* shapes,
                          int64_t* total) {
    PpoLayout L = make_ppo_layout(spec, hs);
    const int n = hs.cat ? L.n - 1 : L.n;
    for (int e = 0; e < n; ++e) {
        const int i = hs.cat ? cat_internal_index(*spec, e) : e;
        if (offsets) offsets[e] = L.off[i];
        if (sizes) sizes[e] = L.size[i];
        if (shapes) { shapes[e * 2] = L.shape[i][0]; shapes[e * 2 + 1] = L.shape[i][1]; }
    }
    if (total) *total = L.total;
    return CPB_OK;
}

static int32_t ppo_forward(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* states,
                           int32_t batch, const float* noise, float* action, float* value, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_forward: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && states && action && value, "ppo_forward: NULL pointer");
    CPB_TRY(run_trunks(spec, L, pl, params, states, nullptr, batch, s));
    HeadArgs h = head_args(spec, hs, L, params, batch);
    h.hp = trunk_buf(pl.h, *spec, 0, spec->num_policy - 1, batch); h.hv = trunk_buf(pl.h, *spec, 1, spec->num_value - 1, batch);
    h.noise = noise; h.action_out = action; h.v_out = value;
    launch_head<2>(hs, batch, h, s);
    CPB_LAUNCHED();
    return CPB_OK;
}

static int32_t ppo_loss_grad(const cpb_ppo_spec* spec, const HeadShape& hs, const float* params, const float* params_old,
                             const float* states, const float* actions, const float* returns, const float* advantages,
                             const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                             int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_loss_grad: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && params_old && states && actions && returns && advantages && grads, "ppo_loss_grad: NULL pointer");
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    CPB_TRY(run_old_logp(spec, hs, L, pl, params_old, states, actions, idx, batch, s));
    return run_loss_grad(spec, hs, L, pl, params, states, actions, returns, advantages, idx, batch, pl.logp_old, 0, grads,
                         metrics, Guards{}, s);
}

static int32_t ppo_train_step(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old,
                              float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                              const float* states, const float* actions, const float* returns, const float* advantages,
                              const int32_t* idx, int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes,
                              void* stream) {
    CPB_REQUIRE(lr_dev != nullptr, "ppo_train_step: lr_dev is NULL");
    CPB_TRY(ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                          workspace, workspace_bytes, stream));
    PpoLayout L = make_ppo_layout(spec, hs);
    return launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f,
                       (cudaStream_t)stream);
}

static int32_t ppo_train_step_opts(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, const float* params_old,
                                   float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                   const float* states, const float* actions, const float* returns,
                                   const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                   const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                   void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(batch >= 1, "ppo_train_step_opts: batch must be >= 1");
    CPB_PPO_PLAN(batch, 0);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                returns && advantages, "ppo_train_step_opts: NULL pointer");
    Guards gd;
    CPB_TRY(make_guards(opts, pl, stop, steps_applied, s, &gd));
    CPB_TRY(launch_fill_zero(grads, L.total, s));
    CPB_TRY(run_old_logp(spec, hs, L, pl, params_old, states, actions, idx, batch, s));
    CPB_TRY(run_loss_grad(spec, hs, L, pl, params, states, actions, returns, advantages, idx, batch, pl.logp_old, 0, grads,
                          metrics, gd, s));
    CPB_TRY(launch_grad_norm(grads, L.total, gd, metrics, s));
    return launch_adam(params, grads, adam_m, adam_v, L.total, adam_powers, 0.f, lr_dev, 0.9f, 0.999f, 1e-8f, s, gd.stop,
                       gd.clip, gd.steps);
}

// learn and its options twin (guarded: opts / steps_applied are used and the metrics rows are 7 wide)
static int32_t ppo_learn(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old, float* grads,
                         float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                         const float* actions, const double* rewards, const double* values, double bootstrap_value,
                         const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                         int32_t batch_size, const int32_t* perms, float* metrics, bool guarded,
                         const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                         int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(T >= 1 && batch_size >= 1 && num_epochs >= 0, "ppo_learn: bad sizes");
    CPB_PPO_PLAN(batch_size < T ? batch_size : T, T);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                rewards && values && dones, "ppo_learn: NULL pointer");
    CPB_REQUIRE(perms != nullptr || num_epochs == 0, "ppo_learn: perms is NULL");
    Guards gd{};
    if (guarded) CPB_TRY(make_guards(opts, pl, nullptr, steps_applied, s, &gd));
    // GAE, returns, normalised advantages (float64), rounded to float32 like the reference's feed
    gae_kernel<<<1, 1024, 0, s>>>(rewards, values, bootstrap_value, dones, T, gamma, lam, nullptr, nullptr, nullptr,
                                  pl.ret32, pl.adv32, pl.gae_scratch);
    CPB_LAUNCHED();
    return learn_update(spec, hs, L, pl, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, T,
                        num_epochs, batch_size, perms, metrics, gd, s);
}

// learn_segments and its options twin
static int32_t ppo_learn_segments(const cpb_ppo_spec* spec, const HeadShape& hs, float* params, float* params_old,
                                  float* grads, float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                  const float* states, const float* actions, const double* rewards,
                                  const double* values, const double* bootstrap_values, const double* dones,
                                  const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                  double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                  float* metrics, bool guarded, const cpb_ppo_learn_options* opts,
                                  int32_t* steps_applied, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_REQUIRE(num_segments >= 1 && rows >= num_segments && batch_size >= 1 && num_epochs >= 0,
                "ppo_learn_segments: bad sizes");
    CPB_PPO_PLAN(batch_size < rows ? batch_size : rows, rows);
    CPB_REQUIRE(params && params_old && grads && adam_m && adam_v && adam_powers && lr_dev && states && actions &&
                rewards && values && bootstrap_values && dones && segment_offsets, "ppo_learn_segments: NULL pointer");
    CPB_REQUIRE(perms != nullptr || num_epochs == 0, "ppo_learn_segments: perms is NULL");
    Guards gd{};
    if (guarded) CPB_TRY(make_guards(opts, pl, nullptr, steps_applied, s, &gd));
    // GAE per segment, then returns and advantages normalised over all rows (float64), rounded to float32
    CPB_TRY(launch_gae_segments(rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                                pl.gae_scratch, nullptr, nullptr, pl.ret32, pl.adv32, s));
    return learn_update(spec, hs, L, pl, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rows,
                        num_epochs, batch_size, perms, metrics, gd, s);
}

extern "C" {

int32_t cpb_ppo_num_tensors(void) { return kLegacyPpoTensors; }
const char* cpb_ppo_tensor_name(int32_t i) {
    cpb_ppo_spec sp;
    memset(&sp, 0, sizeof(sp));
    sp.num_policy = sp.num_value = 2;
    return ppo_tensor_name(&sp, i);
}

int32_t cpb_ppo_spec_num_tensors(const cpb_ppo_spec* spec) {
    CPB_TRY(check_ppo_spec(spec));
    return 2 * (spec->num_policy + spec->num_value) + 5;
}
const char* cpb_ppo_spec_tensor_name(const cpb_ppo_spec* spec, int32_t i) {
    if (check_ppo_spec(spec) != CPB_OK) return nullptr;
    return ppo_tensor_name(spec, i);
}

int32_t cpb_ppo_spec_layout(const cpb_ppo_spec* spec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_TRY(check_ppo_spec(spec));
    return ppo_layout(spec, gauss_head(spec), offsets, sizes, shapes, total);
}

int64_t cpb_ppo_spec_workspace_bytes(const cpb_ppo_spec* spec, int32_t max_batch, int32_t horizon) {
    if (check_ppo_spec(spec) != CPB_OK || max_batch < 1 || horizon < 0) return CPB_ERR_INVALID_ARGUMENT;
    return make_ppo_plan(nullptr, 0, spec, gauss_head(spec), max_batch, horizon).bytes;
}

// the cpb_ppo_spec_* entry points: check the spec, then the shared implementation with the Gaussian head
#define CPB_PPO_GAUSS()              \
    CPB_TRY(check_ppo_spec(spec));   \
    const HeadShape hs = gauss_head(spec);

int32_t cpb_ppo_spec_forward(const cpb_ppo_spec* spec, const float* params, const float* states, int32_t batch,
                             const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                             void* stream) {
    CPB_PPO_GAUSS();
    return ppo_forward(spec, hs, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_loss_grad(const cpb_ppo_spec* spec, const float* params, const float* params_old,
                               const float* states, const float* actions, const float* returns, const float* advantages,
                               const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                         workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_train_step(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                                const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                                int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_train_step(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, returns,
                          advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_train_step_opts(const cpb_ppo_spec* spec, float* params, const float* params_old, float* grads,
                                     float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                     const float* states, const float* actions, const float* returns,
                                     const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                     const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_train_step_opts(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                               returns, advantages, idx, batch, metrics, opts, stop, steps_applied, workspace,
                               workspace_bytes, stream);
}

int32_t cpb_gae(const double* rewards, const double* values, double bootstrap_value, const double* dones, int32_t T,
                double gamma, double lam, double* advantages, double* returns, double* advantages_norm, void* stream) {
    CPB_REQUIRE(rewards && values && dones && T >= 1, "gae: bad arguments");
    CPB_REQUIRE(advantages != nullptr, "gae: advantages output is required");
    gae_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(rewards, values, bootstrap_value, dones, T, gamma, lam, advantages,
                                                      returns, advantages_norm, nullptr, nullptr, nullptr);
    CPB_LAUNCHED();
    return CPB_OK;
}

int32_t cpb_ppo_spec_learn(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, double bootstrap_value,
                           const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                           int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, false, nullptr,
                     nullptr, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_spec_learn_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads, float* adam_m,
                                float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                                const float* actions, const double* rewards, const double* values, double bootstrap_value,
                                const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                                int32_t batch_size, const int32_t* perms, float* metrics,
                                const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                                int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, true, opts,
                     steps_applied, workspace, workspace_bytes, stream);
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

int32_t cpb_ppo_spec_learn_segments(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                    double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                    float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, false, nullptr, nullptr, workspace, workspace_bytes,
                              stream);
}

int32_t cpb_ppo_spec_learn_segments_opts(const cpb_ppo_spec* spec, float* params, float* params_old, float* grads,
                                         float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                         const float* states, const float* actions, const double* rewards,
                                         const double* values, const double* bootstrap_values, const double* dones,
                                         const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                         double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                         float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_GAUSS();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, true, opts, steps_applied, workspace,
                              workspace_bytes, stream);
}

// ---- The categorical twins: check the cpb_ppo_cat_spec, then the shared implementation with its head
#define CPB_PPO_CAT()                 \
    HeadShape hs;                     \
    CPB_TRY(cat_head(cspec, &hs));    \
    const cpb_ppo_spec* spec = &cspec->spec;

int32_t cpb_ppo_cat_num_tensors(const cpb_ppo_cat_spec* cspec) {
    CPB_PPO_CAT();
    return 2 * (spec->num_policy + spec->num_value) + 4;
}
const char* cpb_ppo_cat_tensor_name(const cpb_ppo_cat_spec* cspec, int32_t i) {
    HeadShape hs;
    if (cat_head(cspec, &hs) != CPB_OK) return nullptr;
    const cpb_ppo_spec* spec = &cspec->spec;
    if (i < 0 || i >= 2 * (spec->num_policy + spec->num_value) + 4) return nullptr;
    const int k = cat_internal_index(*spec, i);
    if (k == 2 * spec->num_policy) return "action_logits/kernel";
    if (k == 2 * spec->num_policy + 1) return "action_logits/bias";
    return ppo_tensor_name(spec, k);
}
int32_t cpb_ppo_cat_layout(const cpb_ppo_cat_spec* cspec, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_PPO_CAT();
    return ppo_layout(spec, hs, offsets, sizes, shapes, total);
}
int64_t cpb_ppo_cat_workspace_bytes(const cpb_ppo_cat_spec* cspec, int32_t max_batch, int32_t horizon) {
    HeadShape hs;
    if (cat_head(cspec, &hs) != CPB_OK || max_batch < 1 || horizon < 0) return CPB_ERR_INVALID_ARGUMENT;
    return make_ppo_plan(nullptr, 0, &cspec->spec, hs, max_batch, horizon).bytes;
}

int32_t cpb_ppo_cat_forward(const cpb_ppo_cat_spec* cspec, const float* params, const float* states, int32_t batch,
                            const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                            void* stream) {
    CPB_PPO_CAT();
    return ppo_forward(spec, hs, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_loss_grad(const cpb_ppo_cat_spec* cspec, const float* params, const float* params_old,
                              const float* states, const float* actions, const float* returns, const float* advantages,
                              const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                              int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_loss_grad(spec, hs, params, params_old, states, actions, returns, advantages, idx, batch, grads, metrics,
                         workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_train_step(const cpb_ppo_cat_spec* cspec, float* params, const float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                               int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_train_step(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, returns,
                          advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_train_step_opts(const cpb_ppo_cat_spec* cspec, float* params, const float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const float* returns,
                                    const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                    const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_train_step_opts(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                               returns, advantages, idx, batch, metrics, opts, stop, steps_applied, workspace,
                               workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads, float* adam_m,
                          float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                          const float* actions, const double* rewards, const double* values, double bootstrap_value,
                          const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                          int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, false, nullptr,
                     nullptr, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn_opts(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                               float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const double* rewards, const double* values,
                               double bootstrap_value, const double* dones, int32_t T, double gamma, double lam,
                               int32_t num_epochs, int32_t batch_size, const int32_t* perms, float* metrics,
                               const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions, rewards,
                     values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics, true, opts,
                     steps_applied, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_cat_learn_segments(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                                   float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                   const float* states, const float* actions, const double* rewards,
                                   const double* values, const double* bootstrap_values, const double* dones,
                                   const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                   double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                   float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, false, nullptr, nullptr, workspace, workspace_bytes,
                              stream);
}

int32_t cpb_ppo_cat_learn_segments_opts(const cpb_ppo_cat_spec* cspec, float* params, float* params_old, float* grads,
                                        float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                        const float* states, const float* actions, const double* rewards,
                                        const double* values, const double* bootstrap_values, const double* dones,
                                        const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                        double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                        float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_CAT();
    return ppo_learn_segments(spec, hs, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_values, dones, segment_offsets, num_segments, rows, gamma, lam,
                              num_epochs, batch_size, perms, metrics, true, opts, steps_applied, workspace,
                              workspace_bytes, stream);
}

// ---- The two-per-side entry points: the spec twins at {hidden1, hidden2} / {hidden1, hidden2}
#define CPB_PPO_SPEC_OF(cfg) \
    cpb_ppo_spec spec_;      \
    CPB_TRY(ppo_spec_of(cfg, &spec_));

int32_t cpb_ppo_layout(const cpb_ppo_config* cfg, int64_t* offsets, int64_t* sizes, int32_t* shapes, int64_t* total) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_layout(&spec_, offsets, sizes, shapes, total);
}

int64_t cpb_ppo_workspace_bytes(const cpb_ppo_config* cfg, int32_t max_batch, int32_t horizon) {
    cpb_ppo_spec spec_;
    if (ppo_spec_of(cfg, &spec_) != CPB_OK) return CPB_ERR_INVALID_ARGUMENT;
    return cpb_ppo_spec_workspace_bytes(&spec_, max_batch, horizon);
}

int32_t cpb_ppo_forward(const cpb_ppo_config* cfg, const float* params, const float* states, int32_t batch,
                        const float* noise, float* action, float* value, void* workspace, int64_t workspace_bytes,
                        void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_forward(&spec_, params, states, batch, noise, action, value, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_loss_grad(const cpb_ppo_config* cfg, const float* params, const float* params_old,
                          const float* states, const float* actions, const float* returns, const float* advantages,
                          const int32_t* idx, int32_t batch, float* grads, float* metrics, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_loss_grad(&spec_, params, params_old, states, actions, returns, advantages, idx, batch, grads,
                                  metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_train_step(const cpb_ppo_config* cfg, float* params, const float* params_old, float* grads,
                           float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const float* returns, const float* advantages, const int32_t* idx,
                           int32_t batch, float* metrics, void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_train_step(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                                   returns, advantages, idx, batch, metrics, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_train_step_opts(const cpb_ppo_config* cfg, float* params, const float* params_old, float* grads,
                                float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                const float* states, const float* actions, const float* returns,
                                const float* advantages, const int32_t* idx, int32_t batch, float* metrics,
                                const cpb_ppo_learn_options* opts, uint32_t* stop, int32_t* steps_applied,
                                void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_train_step_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                        actions, returns, advantages, idx, batch, metrics, opts, stop, steps_applied,
                                        workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                      float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                      const float* actions, const double* rewards, const double* values, double bootstrap_value,
                      const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                      int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                      int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                              rewards, values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms, metrics,
                              workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                           float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                           const float* actions, const double* rewards, const double* values, double bootstrap_value,
                           const double* dones, int32_t T, double gamma, double lam, int32_t num_epochs,
                           int32_t batch_size, const int32_t* perms, float* metrics,
                           const cpb_ppo_learn_options* opts, int32_t* steps_applied, void* workspace,
                           int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states, actions,
                                   rewards, values, bootstrap_value, dones, T, gamma, lam, num_epochs, batch_size, perms,
                                   metrics, opts, steps_applied, workspace, workspace_bytes, stream);
}

int32_t cpb_ppo_learn_segments(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads, float* adam_m,
                               float* adam_v, float* adam_powers, const float* lr_dev, const float* states,
                               const float* actions, const double* rewards, const double* values,
                               const double* bootstrap_values, const double* dones, const int32_t* segment_offsets,
                               int32_t num_segments, int32_t rows, double gamma, double lam, int32_t num_epochs,
                               int32_t batch_size, const int32_t* perms, float* metrics, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_segments(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                       actions, rewards, values, bootstrap_values, dones, segment_offsets, num_segments,
                                       rows, gamma, lam, num_epochs, batch_size, perms, metrics, workspace,
                                       workspace_bytes, stream);
}

int32_t cpb_ppo_learn_segments_opts(const cpb_ppo_config* cfg, float* params, float* params_old, float* grads,
                                    float* adam_m, float* adam_v, float* adam_powers, const float* lr_dev,
                                    const float* states, const float* actions, const double* rewards,
                                    const double* values, const double* bootstrap_values, const double* dones,
                                    const int32_t* segment_offsets, int32_t num_segments, int32_t rows, double gamma,
                                    double lam, int32_t num_epochs, int32_t batch_size, const int32_t* perms,
                                    float* metrics, const cpb_ppo_learn_options* opts, int32_t* steps_applied,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
    CPB_PPO_SPEC_OF(cfg);
    return cpb_ppo_spec_learn_segments_opts(&spec_, params, params_old, grads, adam_m, adam_v, adam_powers, lr_dev, states,
                                            actions, rewards, values, bootstrap_values, dones, segment_offsets,
                                            num_segments, rows, gamma, lam, num_epochs, batch_size, perms, metrics, opts,
                                            steps_applied, workspace, workspace_bytes, stream);
}

}  // extern "C"
