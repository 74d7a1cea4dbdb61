// common.cuh -- shared helpers for libctcb200 (H100, sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/ctcb200.h"

namespace ctcb {

extern thread_local char g_last_error[512];
extern std::atomic<uint64_t> g_launch_count;

int set_error(int code, const char *fmt, ...);

inline void count_launch(int n = 1) { g_launch_count.fetch_add((uint64_t)n, std::memory_order_relaxed); }

#define CTCB_CUDA_CHECK(expr)                                                                   \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess)                                                                  \
            return ::ctcb::set_error(CTCB_ECUDA, "%s failed: %s (%s:%d)", #expr,                \
                                     cudaGetErrorString(_e), __FILE__, __LINE__);               \
    } while (0)

#define CTCB_LAUNCH_CHECK()                                                                     \
    do {                                                                                        \
        ::ctcb::count_launch();                                                                 \
        cudaError_t _e = cudaGetLastError();                                                    \
        if (_e != cudaSuccess)                                                                  \
            return ::ctcb::set_error(CTCB_ECUDA, "kernel launch failed: %s (%s:%d)",            \
                                     cudaGetErrorString(_e), __FILE__, __LINE__);               \
    } while (0)

int num_sms();

// Optional per-phase device timing (ctcb_profile_*): CUDA events recorded on the launching stream
// around each phase of the step; off by default so the timed benchmark region carries no events.
struct ProfScope {
    int idx;
    cudaStream_t st;
    ProfScope(const char *name, cudaStream_t s);
    ~ProfScope();
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace ctcb
