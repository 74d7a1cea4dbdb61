// common.cu -- error string, launch counter, device queries.
#include "common.cuh"
#include <stdarg.h>
#include <string.h>
#include <map>
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
    e = cudaGraphInstantiate(&h->exec, g, 0);
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
