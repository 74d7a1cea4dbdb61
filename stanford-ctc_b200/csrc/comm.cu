// comm.cu -- the data-parallel exchange step behind the C ABI: one communicator per process (one process per
// GPU), the flat gradient (+ its 4-float statistics tail) summed over ranks with NCCL over NVLink / NVSwitch.
//
// The reference has no multi-GPU path at all: its only device hook is the CUDA_DEVICE variable
// (ctc_fast/runNNet.py:117-120), and every utterance is a complete optimisation step
// (sgd.py:70-161).  Utterances are independent until the update, so a step's minibatch is sharded over ranks and
// this is the single exchange of the step (SURVEY.md 8b/8e: ctcb_allreduce_grads).
//
// NCCL is resolved at run time (dlopen): a process that already carries a libnccl.so.2 -- PyTorch bundles one --
// keeps using exactly that copy, a plain C/C++ host gets the system library, and libctcb200.so itself has no link
// dependency on NCCL (single-GPU users never load it).
#include "common.cuh"
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>
#include <new>

namespace ctcb {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

static NcclApi &nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {           // a copy the process already loaded (e.g. PyTorch's) wins
        api.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
        if (api.handle) break;
    }
    for (int i = 0; !api.handle && i < 2; ++i) api.handle = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) return api;
#define CTCB_NCCL_SYM(field, sym) *(void **)(&api.field) = dlsym(api.handle, sym)
    CTCB_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
    CTCB_NCCL_SYM(CommInitRank, "ncclCommInitRank");
    CTCB_NCCL_SYM(AllReduce, "ncclAllReduce");
    CTCB_NCCL_SYM(CommDestroy, "ncclCommDestroy");
    CTCB_NCCL_SYM(GroupStart, "ncclGroupStart");
    CTCB_NCCL_SYM(GroupEnd, "ncclGroupEnd");
    CTCB_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef CTCB_NCCL_SYM
    api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.CommDestroy && api.GroupStart && api.GroupEnd &&
             api.GetErrorString;
    return api;
}

#define CTCB_NCCL_CHECK(expr)                                                                                  \
    do {                                                                                                       \
        ncclResult_t _r = (expr);                                                                              \
        if (_r != ncclSuccess)                                                                                 \
            return ::ctcb::set_error(CTCB_ECUDA, "%s failed: %s (%s:%d)", #expr, nccl_api().GetErrorString(_r), \
                                     __FILE__, __LINE__);                                                      \
    } while (0)

}  // namespace ctcb

using namespace ctcb;

struct ctcb_comm {
    ncclComm_t comm;
    int rank, world;
};

static int need_nccl(const char *who) {
    if (!nccl_api().ok) return set_error(CTCB_ECUDA, "%s: libnccl.so.2 could not be loaded (%s)", who, dlerror() ? dlerror() : "missing symbols");
    return CTCB_OK;
}

extern "C" int ctcb_comm_get_unique_id(void *id_out) {
    static_assert(sizeof(ncclUniqueId) == CTCB_COMM_ID_BYTES, "ncclUniqueId size");
    if (!id_out) return set_error(CTCB_EINVAL, "ctcb_comm_get_unique_id: null pointer");
    int rc = need_nccl("ctcb_comm_get_unique_id");
    if (rc != CTCB_OK) return rc;
    CTCB_NCCL_CHECK(nccl_api().GetUniqueId((ncclUniqueId *)id_out));
    return CTCB_OK;
}

extern "C" int ctcb_comm_create(const void *id, int rank, int world, ctcb_comm **out) {
    if (!id || !out || world < 1 || rank < 0 || rank >= world)
        return set_error(CTCB_EINVAL, "ctcb_comm_create: bad arguments (rank %d of %d)", rank, world);
    int rc = need_nccl("ctcb_comm_create");
    if (rc != CTCB_OK) return rc;
    ctcb_comm *c = new (std::nothrow) ctcb_comm;
    if (!c) return set_error(CTCB_ENOMEM, "ctcb_comm_create: out of host memory");
    c->rank = rank;
    c->world = world;
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof(uid));
    ncclResult_t r = nccl_api().CommInitRank(&c->comm, world, uid, rank);     // uses the calling thread's current device
    if (r != ncclSuccess) {
        delete c;
        return set_error(CTCB_ECUDA, "ncclCommInitRank failed: %s", nccl_api().GetErrorString(r));
    }
    *out = c;
    return CTCB_OK;
}

extern "C" void ctcb_comm_destroy(ctcb_comm *c) {
    if (!c) return;
    if (nccl_api().ok) nccl_api().CommDestroy(c->comm);
    delete c;
}

extern "C" int ctcb_comm_rank(const ctcb_comm *c) { return c ? c->rank : -1; }
extern "C" int ctcb_comm_world(const ctcb_comm *c) { return c ? c->world : 0; }

extern "C" int ctcb_allreduce_grads(ctcb_comm *c, float *grads, int64_t n, void *stream) {
    if (!c || !grads || n < 0) return set_error(CTCB_EINVAL, "ctcb_allreduce_grads: bad arguments");
    if (n == 0 || c->world == 1) return CTCB_OK;
    ProfScope ps("allreduce", (cudaStream_t)stream);
    CTCB_NCCL_CHECK(nccl_api().AllReduce(grads, grads, (size_t)n, ncclFloat32, ncclSum, c->comm, (cudaStream_t)stream));
    return CTCB_OK;
}

// Several disjoint ranges in ONE NCCL launch (grouped); used by brnn.cu for the part of the gradient that is not reduced early.
namespace ctcb {
int comm_allreduce_ranges(ctcb_comm *c, float *const *ptrs, const int64_t *counts, int k, cudaStream_t st) {
    if (!c) return set_error(CTCB_EINVAL, "comm_allreduce_ranges: null communicator");
    if (c->world == 1) return CTCB_OK;
    ProfScope ps("allreduce", st);
    CTCB_NCCL_CHECK(nccl_api().GroupStart());
    ncclResult_t bad = ncclSuccess;
    for (int i = 0; i < k; ++i) {
        if (counts[i] <= 0) continue;
        ncclResult_t r = nccl_api().AllReduce(ptrs[i], ptrs[i], (size_t)counts[i], ncclFloat32, ncclSum, c->comm, st);
        if (r != ncclSuccess) bad = r;
    }
    CTCB_NCCL_CHECK(nccl_api().GroupEnd());
    CTCB_NCCL_CHECK(bad);
    return CTCB_OK;
}
int comm_world(const ctcb_comm *c) { return c ? c->world : 1; }
}  // namespace ctcb
