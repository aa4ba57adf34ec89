// Shared helpers for libcarla_ppo_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/carla_ppo_b200.h"

namespace cpb {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern int64_t g_launches;

#define CPB_REQUIRE(cond, ...)                                   \
    do {                                                         \
        if (!(cond)) {                                           \
            cpb::set_error(__VA_ARGS__);                         \
            return CPB_ERR_INVALID_ARGUMENT;                     \
        }                                                        \
    } while (0)

#define CPB_CUDA(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            cpb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                        \
            return CPB_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

// call after every kernel launch
#define CPB_LAUNCHED()                                                                    \
    do {                                                                                  \
        ++cpb::g_launches;                                                                \
        cudaError_t _e = cudaGetLastError();                                              \
        if (_e != cudaSuccess) {                                                          \
            cpb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),    \
                           __FILE__, __LINE__);                                           \
            return CPB_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

#define CPB_TRY(expr)                 \
    do {                              \
        int32_t _s = (expr);          \
        if (_s != CPB_OK) return _s;  \
    } while (0)

// ---- optional per-call-site timing (see cpb_profile_* in the header) ---------------------------
extern bool g_profile_on;
void profile_begin(const char* label, cudaStream_t s);
void profile_end(cudaStream_t s);
struct ProfScope {
    cudaStream_t s;
    bool on;
    ProfScope(const char* label, cudaStream_t stream) : s(stream), on(g_profile_on) {
        if (on) profile_begin(label, s);
    }
    ~ProfScope() {
        if (on) profile_end(s);
    }
};

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// The tensor-core kernels (tc_tapgemm, tc_wgrad) address an activation tensor of `batch` images of `img` floats with
// 32-bit offsets.  Their launchers refuse a problem outside this rule; the ConvVAE planner derives its batch bound from it.
static inline bool tc_offsets_fit(int64_t batch, int64_t img) { return batch * img < (1ll << 31); }
static inline int64_t tc_max_batch(int64_t img) { return ((1ll << 31) - 1) / img; }

// ---- workspace bump allocator ---------------------------------------------------------------
struct Arena {
    char* base;
    int64_t cap;
    int64_t off;
    bool overflow;
    Arena(void* p, int64_t bytes) : base((char*)p), cap(bytes), off(0), overflow(false) {}
    template <typename T>
    T* take(int64_t count) {
        int64_t bytes = align_up(count * (int64_t)sizeof(T), 256);
        T* r = (T*)(base + off);
        off += bytes;
        if (off > cap) overflow = true;
        return r;
    }
};

// ---- device helpers -------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif

}  // namespace cpb
