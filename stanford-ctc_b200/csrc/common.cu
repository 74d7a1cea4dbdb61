// common.cu -- error string, launch counter, device queries, planner knobs.
#include "common.cuh"
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

namespace ctcb {
thread_local char g_last_error[512] = "";
std::atomic<uint64_t> g_launch_count{0};

int set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
    return code;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
    }
    return n;
}

size_t max_smem_optin() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
            cudaGetLastError();
            return 232448;
        }
    }
    return (size_t)n;
}

static void stream_priority_range(int *least, int *greatest) {
    static int lo = 0, hi = 0;
    static bool read = false;
    if (!read) {
        if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) { cudaGetLastError(); lo = hi = 0; }
        read = true;
    }
    *least = lo;
    *greatest = hi;
}
int stream_priority_least() { int lo, hi; stream_priority_range(&lo, &hi); return lo; }
int stream_priority_greatest() { int lo, hi; stream_priority_range(&lo, &hi); return hi; }

// The documented values of each knob, in the order of enum Knob: the string values[v] sets the value v, and where
// count > 0 the decimal numbers 1..count set themselves.  A value the environment gives that is not listed here leaves
// the default in effect.
struct KnobDef { const char *name; int dflt; const char *values[9]; int count; };
static const KnobDef KNOBS[KNOB_COUNT] = {
    {"CTCB_GEMM", 0, {nullptr, "simt"}},
    {"CTCB_GEMM_TC_COPY", 0, {"0", "1"}},
    {"CTCB_GEMM_TRACE", 0, {nullptr, "1"}},
    {"CTCB_SWEEP", 0, {"auto", "barrier", "reread"}},
    {"CTCB_SWEEP_NB", 0, {nullptr, "1", "2", "3", "4", "5", "6", "7", "8"}},
    {"CTCB_SWEEP_TC", 1, {"0", "1", "2"}},
    {"CTCB_SWEEP_TC_CS", 4, {nullptr, "1", "2", nullptr, "4"}},
    {"CTCB_SWEEP_TC_COOP", 1, {"0"}},
    {"CTCB_SWEEP_TRACE", 0, {nullptr, "1"}},
    {"CTCB_CTC", 0, {"auto", "warp", "pair", "par", "ckpt"}},
    {"CTCB_LSTM", 0, {"auto", "reread"}},
    {"CTCB_LSTM_PARTS", 0, {"auto"}, COOP_SWEEP_MAX_PARTS},
    {"CTCB_SWEEP_PARTS", 0, {"auto"}, COOP_SWEEP_MAX_PARTS},
    {"CTCB_STALL", STALL_OFF, {"off", "main", "side"}},
    {"CTCB_STALL_US", 2000, {}, STALL_MAX_US},
};
static int g_knob_initial[KNOB_COUNT], g_knob[KNOB_COUNT];     // what the environment said, what is in effect
static std::once_flag g_knob_once;

static int parse_knob(const KnobDef &d, const char *s) {
    for (int v = 0; v < 9; ++v)
        if (d.values[v] && strcmp(d.values[v], s) == 0) return v;
    if (d.count > 0 && s[0] >= '1' && s[0] <= '9' && strlen(s) <= 9) {
        int v = 0;
        for (const char *c = s; *c; ++c) {
            if (*c < '0' || *c > '9') return -1;
            v = 10 * v + (*c - '0');
        }
        if (v <= d.count) return v;
    }
    return -1;
}

static int *knob_table() {
    std::call_once(g_knob_once, [] {
        for (int k = 0; k < KNOB_COUNT; ++k) {
            const char *e = getenv(KNOBS[k].name);
            const int v = e ? parse_knob(KNOBS[k], e) : -1;
            g_knob_initial[k] = g_knob[k] = v < 0 ? KNOBS[k].dflt : v;
        }
    });
    return g_knob;
}

int knob(Knob k) { return knob_table()[k]; }

static thread_local int g_tf32 = 0;
int tf32_mode() { return g_tf32; }
Tf32Scope::Tf32Scope(int on) : prev(g_tf32) { g_tf32 = on ? 1 : 0; }
Tf32Scope::~Tf32Scope() { g_tf32 = prev; }

// One warp sleeping on %globaltimer until ns have passed; it writes nothing, and ns is clamped to the knob's maximum,
// so the wait always ends.
__global__ void stall_kernel(uint64_t ns) {
    ns = ns < (uint64_t)STALL_MAX_US * 1000u ? ns : (uint64_t)STALL_MAX_US * 1000u;
    uint64_t t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do {
        __nanosleep(1000);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    } while (t - t0 < ns);
}

int stall(cudaStream_t st, int which) {
    if (which == STALL_OFF || knob(KNOB_STALL) != which) return CTCB_OK;
    stall_kernel<<<1, 32, 0, st>>>((uint64_t)knob(KNOB_STALL_US) * 1000u);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

static bool g_prof_on = false;
struct ProfRec { std::string name; cudaEvent_t a, b; };
static std::vector<ProfRec> g_prof;

ProfScope::ProfScope(const char *name, cudaStream_t s) : idx(-1), st(s) {
    if (!g_prof_on) return;
    ProfRec r;
    r.name = name;
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    cudaEventRecord(r.a, s);
    g_prof.push_back(r);
    idx = (int)g_prof.size() - 1;
}
ProfScope::~ProfScope() {
    if (idx >= 0) cudaEventRecord(g_prof[idx].b, st);
}
}  // namespace ctcb

extern "C" void ctcb_profile_enable(int on) { ctcb::g_prof_on = (on != 0); }

extern "C" int ctcb_profile_report(char *buf, size_t cap) {
    using namespace ctcb;
    if (!buf || cap == 0) return set_error(CTCB_EINVAL, "ctcb_profile_report: no buffer");
    if (cudaDeviceSynchronize() != cudaSuccess) return set_error(CTCB_ECUDA, "ctcb_profile_report: sync failed");
    std::map<std::string, std::pair<int, double>> agg;
    for (auto &r : g_prof) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
            auto &e = agg[r.name];
            e.first += 1;
            e.second += ms;
        }
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
    }
    g_prof.clear();
    std::string out = "{";
    bool first = true;
    for (auto &kv : agg) {
        char tmp[256];
        snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"count\": %d, \"total_ms\": %.6f}", first ? "" : ", ",
                 kv.first.c_str(), kv.second.first, kv.second.second);
        out += tmp;
        first = false;
    }
    out += "}";
    if (out.size() + 1 > cap) return set_error(CTCB_ENOMEM, "ctcb_profile_report: buffer too small");
    memcpy(buf, out.c_str(), out.size() + 1);
    return CTCB_OK;
}

extern "C" int ctcb_version(void) { return 100; }
extern "C" const char *ctcb_last_error(void) { return ctcb::g_last_error; }
extern "C" uint64_t ctcb_launch_count(void) { return ctcb::g_launch_count.load(); }

extern "C" int ctcb_debug_set_knob(const char *name, const char *value) {
    using namespace ctcb;
    int *table = knob_table();
    for (int k = 0; name && k < KNOB_COUNT; ++k) {
        if (strcmp(name, KNOBS[k].name) != 0) continue;
        const int v = value ? parse_knob(KNOBS[k], value) : g_knob_initial[k];
        if (v < 0) return set_error(CTCB_EINVAL, "ctcb_debug_set_knob: \"%s\" is not a value of %s", value, name);
        table[k] = v;
        return CTCB_OK;
    }
    return set_error(CTCB_EINVAL, "ctcb_debug_set_knob: unknown knob %s", name ? name : "(null)");
}

extern "C" int ctcb_debug_set_ctc_kernel(int shape) {
    using namespace ctcb;
    if (shape < 0 || shape > 4) return set_error(CTCB_EINVAL, "ctcb_debug_set_ctc_kernel: shape %d not in 0..4", shape);
    knob_table()[KNOB_CTC] = shape;
    return CTCB_OK;
}

// ---- CUDA graphs: one optimisation step (dozens of small launches on two streams) replayed as ONE graph launch ----
struct ctcb_graph {
    cudaGraphExec_t exec;
    uint64_t launches;     // kernels the captured region launched (ctcb_launch_count stays meaningful under replay)
};
static thread_local uint64_t g_capture_launch0 = 0;

extern "C" int ctcb_graph_capture_begin(void *stream) {
    using namespace ctcb;
    // ThreadLocal: other threads of the host program (loaders, other GPUs' drivers) stay free to call CUDA
    CTCB_CUDA_CHECK(cudaStreamBeginCapture((cudaStream_t)stream, cudaStreamCaptureModeThreadLocal));
    g_capture_launch0 = g_launch_count.load();
    return CTCB_OK;
}

extern "C" int ctcb_graph_capture_end(void *stream, ctcb_graph **out) {
    using namespace ctcb;
    if (!out) return set_error(CTCB_EINVAL, "ctcb_graph_capture_end: null output");
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture((cudaStream_t)stream, &g);
    if (e != cudaSuccess || !g) {
        cudaGetLastError();
        return set_error(CTCB_ECUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
    }
    ctcb_graph *h = new (std::nothrow) ctcb_graph;
    if (!h) { cudaGraphDestroy(g); return set_error(CTCB_ENOMEM, "ctcb_graph_capture_end: out of host memory"); }
    h->launches = g_launch_count.load() - g_capture_launch0;
    g_launch_count.fetch_sub(h->launches);      // nothing ran during capture
    // per-node priorities: without the flag every node runs at the launching stream's priority, and the BPTT sweep
    // would no longer take its SMs ahead of the side stream's weight gradients (brnn.cu)
    e = cudaGraphInstantiateWithFlags(&h->exec, g, cudaGraphInstantiateFlagUseNodePriority);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) {
        delete h;
        return set_error(CTCB_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
    }
    *out = h;
    return CTCB_OK;
}

extern "C" int ctcb_graph_launch(ctcb_graph *h, void *stream) {
    using namespace ctcb;
    if (!h) return set_error(CTCB_EINVAL, "ctcb_graph_launch: null graph");
    CTCB_CUDA_CHECK(cudaGraphLaunch(h->exec, (cudaStream_t)stream));
    count_launch((int)h->launches);
    return CTCB_OK;
}

extern "C" void ctcb_graph_destroy(ctcb_graph *h) {
    if (!h) return;
    cudaGraphExecDestroy(h->exec);
    delete h;
}
