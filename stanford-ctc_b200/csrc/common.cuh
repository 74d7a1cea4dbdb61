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
// The most dynamic shared memory one CTA can opt in to (cudaDevAttrMaxSharedMemoryPerBlockOptin).  A planner refuses a
// footprint above it with CTCB_EINVAL before it asks for the kernel attribute, whose failure is a CUDA error.
size_t max_smem_optin();
// The device's stream priority range (cudaDeviceGetStreamPriorityRange): least is the default, greatest runs first.
int stream_priority_least();
int stream_priority_greatest();

// Debug / measurement overrides of the planners (INTEGRATION.md section 4): one table (common.cu), filled from the
// environment at first use and changed by ctcb_debug_set_knob.  Planners read it through knob() on every planning call.
enum Knob { KNOB_GEMM, KNOB_GEMM_TC_COPY, KNOB_GEMM_TRACE, KNOB_SWEEP, KNOB_SWEEP_NB, KNOB_SWEEP_TC, KNOB_SWEEP_TC_CS,
            KNOB_SWEEP_TC_COOP, KNOB_SWEEP_TRACE, KNOB_CTC, KNOB_LSTM, KNOB_LSTM_PARTS, KNOB_SWEEP_PARTS, KNOB_STALL,
            KNOB_STALL_US, KNOB_COUNT };
int knob(Knob k);
// TF32 mode (include/ctcb200.h: ctcb_brnn_config.tf32): the tensor-core contraction and sweep planners take the TF32
// kernels while a Tf32Scope(1) is alive on the calling thread.  A net's calls and the *_tf32 entry points open one
// around their launches; everything else plans the fp32-faithful kernels.
int tf32_mode();
struct Tf32Scope {
    int prev;
    explicit Tf32Scope(int on);
    ~Tf32Scope();
};
// The schedule test's stall hook (CTCB_STALL, CTCB_STALL_US): stall(st, which) launches one warp that holds `st` for
// CTCB_STALL_US microseconds when CTCB_STALL names `which`, and does nothing otherwise (off, the default, names neither).
// The training step calls it right after each point where one of its streams releases or is released by the other.
enum { STALL_OFF = 0, STALL_MAIN = 1, STALL_SIDE = 2 };
constexpr int STALL_MAX_US = 100000;
int stall(cudaStream_t st, int which);
// The most utterance partitions of a cooperative sweep (the generic and LSTM kernels, coop_sweep.cuh): their barrier
// counters ([ndir][parts] words) share 4 KB of scratch with the 16 error words.  CTCB_SWEEP_PARTS and CTCB_LSTM_PARTS
// take auto or 1..COOP_SWEEP_MAX_PARTS.
constexpr int COOP_SWEEP_MAX_PARTS = 500;

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

// What run_sweep launches for (H, B, ndir) under the environment knobs in effect.  One function, select_sweep (sweep.cu),
// makes the choice for the launch, ctcb_debug_sweep_plan and ctcb_sweep_uses_tensor_cores alike.
enum { SWEEP_GENERIC = 0, SWEEP_CLUSTER = 1, SWEEP_TC = 2 };
struct SweepPlan {
    int kernel;             // SWEEP_GENERIC (sweep.cu), SWEEP_CLUSTER (sweep_cluster.cu), SWEEP_TC (sweep_tc.cu)
    int KI;                 // generic / cluster: H / 32 with the weights in registers; 0: weights re-read (generic)
    int cs;                 // tensor-core: K-slices per cluster; cluster: CTAs per cluster (H / 64); generic: 0
    int groups;             // tensor-core: utterance splits (NS); cluster: utterances per cluster (NB); generic: partitions
    int np;                 // tensor-core: utterances per split, the wgmma N
    int stages;             // tensor-core: operand ring stages
    int partial_own;        // tensor-core: 1 when the partial product has a shared-memory region of its own
    uint32_t stage_bytes;   // tensor-core: bytes per ring stage
    size_t smem;            // dynamic shared memory per CTA
    int per_sm;             // generic: CTAs of the kernel one SM holds
    int tf32;               // tensor-core: TF32 mode (tf32_mode() when planned)
};
int select_sweep(int H, int B, int ndir, SweepPlan *p);

// How ctcb_gemm_f32 runs a contraction on the FFMA kernel (gemm_simt.cu); gemm_simt_plan decides it for the launch and
// ctcb_debug_gemm_plan alike.
struct GemmSimtPlan {
    int splits;             // K splits (gridDim.z); > 1 writes partials to the workspace and adds a reduce
    int k_per_split;        // k per split, a multiple of the 16-deep k-tile: the length of each accumulator chain
    int vec;                // 16-byte operand loads (both pitches multiples of 4 floats, both bases 16-byte aligned)
    int ctas;               // CTAs of the launch
};
void gemm_simt_plan(int M, int N, int K, const float *A, int64_t lda, const float *B, int64_t ldb, size_t ws_bytes,
                    GemmSimtPlan *p);
// Both contraction kernels put 128-row output tiles on gridDim.y (at most 65,535): the largest M they take.
constexpr int GEMM_MAX_M = 128 * 65535;

// The zoneout settings of one LSTM sweep launch (include/ctcb200.h: zoneout = 1); run_lstm_sweep (sweep_lstm.cu) takes
// a null pointer for the cell without zoneout.
struct LstmZoneout {
    float zc, zh;
    bool train;                // masks drawn from (seed, *step, g, t, layer, dir, j); else the expectation, lambda = z
    uint64_t seed;
    const int64_t *step;       // device counter, read by the kernel (training mode)
    int64_t first, stride;     // utterance b of the call is minibatch utterance first + stride b
    int layer;                 // hidden-layer index of the temporal layer, 1..255
    float *dhc;                // BPTT: the [ndir][B][H] dh carry
};

}  // namespace ctcb
