// brnn.cu -- batched costAndGrad of the bi-directional recurrent network, orchestrated on one stream.
//
// Replaces nnets.brnnet.NNet.costAndGrad (ctc_fast/nnets/brnnet.py:117-249), which
// runs one utterance at a time as ~8(T-1)+12N+40 cudamat launches with a blocking D2H/H2D round
// trip through the CPU CTC in the middle.  Here a whole minibatch of utterances is one pass:
//
//   layout   : every activation is time-major [T][B][n] fp32 -- one time step of all utterances is a
//              contiguous (B x n) slab, so the layer contractions are single GEMMs over R = T*B rows
//              and the recurrences are (B x H)(H x H) products per step.
//   forward  : per layer one GEMM with bias(+ReLU) fused in the epilogue (brnnet.py:140-141,155-157);
//              each temporal layer (numTemporal of them, stacked) adds the persistent two-direction sweep
//              (sweep.cu) with its own recurrent matrices and For+Back.
//   CTC      : softmax + alpha/beta + gradient in one kernel on the device (ctc.cu); nothing leaves HBM.
//   backward : per layer dW = delta^T X (split-K GEMM over R), db = column sums, delta <- delta W with
//              the ReLU mask fused (brnnet.py:196-204,235-237); BPTT sweep; the recurrent weight
//              gradients are two GEMMs over time-shifted views (brnnet.py:227-230).
// Gradients of the utterances of the batch are summed (the reference never normalises, cf.
// ctc/nnet.py:193-195); a skipped utterance contributes nothing.
#include "common.cuh"
#include <new>

namespace ctcb {
int run_sweep(int mode, int T, int B, int H, const int32_t *Tlen, const float *pre, const float *Wf,
              const float *Wb, float *outF, float *outB, const float *actF, const float *actB, float maxAct,
              unsigned int *counters, void *ws, size_t ws_bytes, cudaStream_t st);
size_t sweep_tc_workspace_bytes(int H, int B);
int run_add2(const float *x, const float *y, float *z, int64_t n, cudaStream_t st);
int run_sumsq(const float *g, int64_t n, float *out, float scale, int accumulate, void *scratch, cudaStream_t st);
int comm_allreduce_ranges(ctcb_comm *c, float *const *ptrs, const int64_t *counts, int k, cudaStream_t st);
int comm_world(const ctcb_comm *c);

// ---- small kernels ---------------------------------------------------------------------------
// column sums of a row-major R x N matrix: stage 1 partials over row blocks, stage 2 final
constexpr int CS_ROWS = 1024;
__global__ void colsum_stage1(const float *__restrict__ x, int64_t R, int N, float *__restrict__ partial) {
    __shared__ float sh[8][33];
    const int n = blockIdx.x * 32 + threadIdx.x;
    const int64_t r0 = (int64_t)blockIdx.y * CS_ROWS;
    const int64_t r1 = (r0 + CS_ROWS < R) ? r0 + CS_ROWS : R;
    float s = 0.f;
    if (n < N)
        for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += x[r * N + n];
    sh[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sh[i][threadIdx.x];
        partial[(int64_t)blockIdx.y * N + n] = t;
    }
}
// the same for row pitches that are a multiple of 4 floats: a block walks FULL-WIDTH row segments (each thread a float4
// column group), so consecutive warps read consecutive 512-byte pieces of a row instead of 128-byte strips 8 KB apart
constexpr int CS_ROWS_MIN = 128;
__global__ void colsum_stage1_wide(const float4 *__restrict__ x, int64_t R, int N4, int rows_per_block, float4 *__restrict__ partial) {
    const int c4 = blockIdx.x * blockDim.x + threadIdx.x;
    if (c4 >= N4) return;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
    const int64_t r1 = (r0 + rows_per_block < R) ? r0 + rows_per_block : R;
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
    int64_t r = r0;
    for (; r + 4 <= r1; r += 4) {
        const float4 v0 = __ldg(x + r * N4 + c4), v1 = __ldg(x + (r + 1) * N4 + c4);
        const float4 v2 = __ldg(x + (r + 2) * N4 + c4), v3 = __ldg(x + (r + 3) * N4 + c4);
        a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
        a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
        a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;
        a3.x += v3.x; a3.y += v3.y; a3.z += v3.z; a3.w += v3.w;
    }
    for (; r < r1; ++r) {
        const float4 v = __ldg(x + r * N4 + c4);
        a0.x += v.x; a0.y += v.y; a0.z += v.z; a0.w += v.w;
    }
    partial[(int64_t)blockIdx.y * N4 + c4] = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y),
                                                        (a0.z + a1.z) + (a2.z + a3.z), (a0.w + a1.w) + (a2.w + a3.w));
}
// ACC: add the column sums into `out` (a later micro-batch of a step) instead of overwriting it
template <bool ACC>
__global__ void colsum_stage2(const float *__restrict__ partial, int nblk, int N, float *__restrict__ out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float s = 0.f;
    for (int i = 0; i < nblk; ++i) s += partial[(int64_t)i * N + n];
    if (ACC) s += out[n];
    out[n] = s;
}

// row softmax of a row-major R x K matrix (forward-only mode, brnnet.py:161-173); one warp per row
__global__ void softmax_rows_kernel(const float *__restrict__ x, float *__restrict__ p, int64_t R, int K) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= R) return;
    const float *xr = x + row * K;
    float m = -3.4e38f;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, xr[k]);
    m = warp_max(m);
    float z = 0.f;
    for (int k = lane; k < K; k += 32) z += expf(xr[k] - m);
    z = warp_sum(z);
    const float inv = 1.f / z;
    for (int k = lane; k < K; k += 32) p[row * K + k] = expf(xr[k] - m) * inv;
}

__global__ void set_scalar_kernel(float *p, float v) { *p = v; }

// stats = {#non-skipped, sum of their nll, #skipped, sweep error flag}; one warp.  The flag rides in the data-parallel
// all-reduce with the rest of the tail, so a wait timeout on one rank is seen (non-zero) by every rank.
// ACC: add into the tail of the earlier micro-batches of the step; the flag only grows, so it stays non-zero.
template <bool ACC>
__global__ void batch_stats_kernel(const float *__restrict__ cost, const int32_t *__restrict__ skip, int B, float *stats,
                                   const unsigned int *__restrict__ errflag) {
    float nv = 0.f, cs = 0.f, ns = 0.f;
    for (int u = threadIdx.x; u < B; u += 32) {
        if (skip[u]) ns += 1.f;
        else { nv += 1.f; cs += cost[u]; }
    }
    nv = warp_sum(nv); cs = warp_sum(cs); ns = warp_sum(ns);
    if (threadIdx.x == 0) {
        float ef = (float)errflag[0];
        if (ACC) { nv += stats[0]; cs += stats[1]; ns += stats[2]; ef += stats[3]; }
        stats[0] = nv; stats[1] = cs; stats[2] = ns; stats[3] = ef;
    }
}

}  // namespace ctcb

using namespace ctcb;

namespace {
// The buffers of a forward-only call: affine map i writes slab i % 2 and reads the other one (or For, the output of
// the uni-directional temporal layer), so two slabs of the wider of H and K carry the whole stack.
struct FwdLayout {
    size_t slab[2];
    size_t For, Back, gemm, gemm_bytes, counters, sweep, sweep_bytes;
    size_t total;
};
}  // namespace

struct ctcb_brnn {
    ctcb_brnn_config cfg;
    int nlayers;        // N + 1 affine maps
    int tl;             // lowest temporal layer or 0
    int nt;             // temporal layers tl .. tl+nt-1 (0 without)
    int sizes[66];      // [D, H.., K]
    // weight/bias gradients of the layers at and above the temporal layer depend only on their delta, so they
    // run on a side stream next to the (latency-bound, 112-SM) BPTT sweep; created on first use
    cudaStream_t side;
    cudaEvent_t ev_delta[66];
    cudaEvent_t ev_side;
    // the two dFor/dBack pairs that stacked temporal layers alternate: ev_pair[p] is recorded on the side stream after
    // its last read of pair p, and the BPTT sweep that writes pair p next waits for it
    cudaEvent_t ev_pair[2];
    bool side_ready;
    // data-parallel callers sum the gradient over ranks first and add reg*W ONCE afterwards (ctcb_brnn_apply_l2_f32);
    // the L2 cost is still reported by every call
    bool defer_l2;
    // data-parallel exchange inside the step (ctcb_brnn_set_comm): the gradients of the layers at and above the temporal
    // layer are summed over ranks on the side stream WHILE the BPTT sweep runs, the rest (+ statistics tail) at the end
    ctcb_comm *comm;
    // the forward layout, computed on the first forward-only call (its GEMM area takes a few hundred size queries)
    bool fwd_ready;
    FwdLayout fwd;
};

static int valid_cfg(const ctcb_brnn_config *c) {
    if (!c) return 0;
    if (c->inputDim <= 0 || c->outputDim <= 1 || c->layerSize <= 0) return 0;
    if (c->numLayers < 1 || c->numLayers > 64) return 0;
    if (c->maxT <= 0 || c->maxB <= 0 || c->maxLabels < 0) return 0;
    if (c->maxLabels > CTCB_CTC_MAX_LABELS) return 0;   // the CTC kernel's register-resident trellis (ctc.cu)
    if (c->numTemporal < 0) return 0;
    // a stacked block must lie inside the hidden layers; k <= 1 keeps the silent "no temporal layer" rule below
    if (c->numTemporal > 1 && (c->temporalLayer <= 0 || c->temporalLayer + c->numTemporal - 1 > c->numLayers)) return 0;
    return 1;
}
static int eff_tl(const ctcb_brnn_config *c) {
    return (c->temporalLayer <= 0 || c->temporalLayer > c->numLayers) ? 0 : c->temporalLayer;
}
// number of temporal layers of a valid config
static int eff_nt(const ctcb_brnn_config *c) {
    if (!eff_tl(c)) return 0;
    return c->numTemporal > 1 ? c->numTemporal : 1;
}
// flat-vector index of the (forward) recurrent matrix of temporal layer j (0-based within the block); the backward
// one, when bi-directional, is two tensors behind it
static int rec_index(const ctcb_brnn_config *c, int j) {
    return 2 * (c->numLayers + 1) + j * (c->unidirectional ? 2 : 4);
}
static void layer_sizes(const ctcb_brnn_config *c, int *sizes) {
    sizes[0] = c->inputDim;
    for (int i = 1; i <= c->numLayers; ++i) sizes[i] = c->layerSize;
    sizes[c->numLayers + 1] = c->outputDim;
}

extern "C" int ctcb_brnn_num_tensors(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    return 2 * (cfg->numLayers + 1) + eff_nt(cfg) * (cfg->unidirectional ? 2 : 4);
}

extern "C" int ctcb_brnn_tensor_info(const ctcb_brnn_config *cfg, int idx, int64_t *offset, int32_t *rows, int32_t *cols) {
    if (!valid_cfg(cfg)) return set_error(CTCB_EINVAL, "ctcb_brnn_tensor_info: bad config");
    const int nt = ctcb_brnn_num_tensors(cfg);
    if (idx < 0 || idx >= nt) return set_error(CTCB_EINVAL, "ctcb_brnn_tensor_info: index %d out of range", idx);
    int sizes[66];
    layer_sizes(cfg, sizes);
    int64_t off = 0;
    for (int t = 0; t < nt; ++t) {
        int r, c;
        const int nl = cfg->numLayers + 1;
        if (t < 2 * nl) {
            const int i = t / 2;
            if (t % 2 == 0) { r = sizes[i + 1]; c = sizes[i]; }
            else { r = sizes[i + 1]; c = 1; }
        } else {
            if ((t - 2 * nl) % 2 == 0) { r = cfg->layerSize; c = cfg->layerSize; }
            else { r = 1; c = 1; }   // the reference's `dummy` bias (brnnet.py:60-72)
        }
        if (t == idx) {
            if (offset) *offset = off;
            if (rows) *rows = r;
            if (cols) *cols = c;
            return CTCB_OK;
        }
        off += (int64_t)r * c;
        off = (off + 3) / 4 * 4;   // keep every tensor 16-byte aligned
    }
    return CTCB_EINVAL;
}

extern "C" int64_t ctcb_brnn_param_count(const ctcb_brnn_config *cfg) {
    const int nt = ctcb_brnn_num_tensors(cfg);
    if (nt == 0) return 0;
    int64_t off; int32_t r, c;
    ctcb_brnn_tensor_info(cfg, nt - 1, &off, &r, &c);
    return (off + (int64_t)r * c + 3) / 4 * 4;
}

namespace {
struct WsLayout {
    size_t X[66];       // X[1..N] activations, X[N+1] logits
    size_t For, Back, dFor, dBack;
    // stacked temporal layers: For / Back of temporal layer j (ForJ[0] = For, BackJ[0] = Back) and the second
    // dFor / dBack pair, which layers of odd j use (0 where not laid out)
    size_t ForJ[64], BackJ[64], dFor2, dBack2;
    size_t D[67];       // D[j]: gradient w.r.t. the output of affine map j (1..N+1)
    size_t gemm2, colsum2;
    size_t ctc, gemm, colsum, scratch, counters, sweep, sweep_bytes, lens_dummy;
    size_t total;
};

WsLayout ws_layout(const ctcb_brnn_config *c) {
    WsLayout w{};
    int sizes[66];
    layer_sizes(c, sizes);
    const size_t R = (size_t)c->maxT * c->maxB;
    const int N = c->numLayers, H = c->layerSize, K = c->outputDim;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    for (int i = 1; i <= N + 1; ++i) w.X[i] = take(R * sizes[i] * sizeof(float));
    if (eff_tl(c)) {
        w.For = take(R * H * sizeof(float));
        w.Back = take(R * H * sizeof(float));
        w.dFor = take(R * H * sizeof(float));
        w.dBack = take(R * H * sizeof(float));
        w.ForJ[0] = w.For;
        w.BackJ[0] = w.Back;
    }
    // every further temporal layer keeps its own For (and Back): the BPTT masks and the recurrent weight gradients
    // read them.  The dFor / dBack pairs alternate between consecutive layers, so a stack needs one more pair.
    const int nt = eff_nt(c);
    const bool uni = (c->unidirectional != 0);
    for (int j = 1; j < nt; ++j) {
        w.ForJ[j] = take(R * H * sizeof(float));
        if (!uni) w.BackJ[j] = take(R * H * sizeof(float));
    }
    if (nt > 1) {
        w.dFor2 = take(R * H * sizeof(float));
        if (!uni) w.dBack2 = take(R * H * sizeof(float));
    }
    const size_t wide = (size_t)(H > K ? H : K);
    for (int j = 1; j <= N + 1; ++j) w.D[j] = take(R * wide * sizeof(float));
    w.ctc = take(ctcb_ctc_workspace_bytes(c->maxB, c->maxT, c->maxLabels));
    size_t g = 0;
    const int Rint = (int)((R > 0x7fffffff) ? 0x7fffffff : R);
    auto need = [&](int M_, int N_, int K_) { size_t b = ctcb_gemm_workspace_bytes(M_, N_, K_); if (b > g) g = b; };
    for (int i = 0; i <= N; ++i) {
        need(Rint, sizes[i + 1], sizes[i]);      // forward   X_i . W^T
        need(Rint, sizes[i], sizes[i + 1]);      // backward  delta . W
        need(sizes[i + 1], sizes[i], Rint);      // weights   delta^T . X_i
    }
    {                                            // recurrent weight gradients (a pair for the bi-directional layer)
        const size_t b = ctcb_gemm_pair_workspace_bytes(H, H, Rint);
        if (b > g) g = b;
    }
    w.gemm = take(g);
    w.gemm2 = take(g);
    w.colsum = take(((R + CS_ROWS_MIN - 1) / CS_ROWS_MIN) * wide * sizeof(float));
    w.colsum2 = take(((R + CS_ROWS_MIN - 1) / CS_ROWS_MIN) * wide * sizeof(float));
    w.scratch = take(8192);
    w.counters = take(sizeof(unsigned int) * 1024);
    w.sweep_bytes = eff_tl(c) ? sweep_tc_workspace_bytes(H, c->maxB) : 0;
    w.sweep = take(w.sweep_bytes);
    w.total = off;
    return w;
}

// Rows per output tile of both contraction kernels (BM of gemm_simt.cu, TC_BM of gemm_tc.cu): their workspace needs
// change with the row count only at multiples of it.
constexpr int GEMM_ROW_TILE = 128;

FwdLayout fwd_layout(const ctcb_brnn_config *c) {
    FwdLayout f{};
    int sizes[66];
    layer_sizes(c, sizes);
    const size_t R = (size_t)c->maxT * c->maxB;
    const int N = c->numLayers, H = c->layerSize, K = c->outputDim;
    const size_t wide = (size_t)(H > K ? H : K);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    f.slab[0] = take(R * wide * sizeof(float));
    f.slab[1] = take(R * wide * sizeof(float));
    if (eff_tl(c)) {
        f.For = take(R * H * sizeof(float));
        if (!c->unidirectional) f.Back = take(R * H * sizeof(float));
    }
    // ctcb_gemm_f32 takes a smaller plan when its area is short of ctcb_gemm_workspace_bytes(R, ..), and that need is
    // not monotone in R = Tmax*B: below one wave of output tiles the tensor-core plan adds split-K partials.  So that a
    // forward contraction takes, at every R <= maxT*maxB, the plan it takes in the training layout, the area is the
    // largest forward need over all such R, capped at the training area (a contraction that falls back there must
    // fall back here too).  The need changes with R only at multiples of the row tile and grows with R once
    // num_sms() row tiles are exceeded (the split counts are then fixed), so those multiples and R itself bound it.
    size_t g = 0;
    const int Rint = (int)((R > 0x7fffffff) ? 0x7fffffff : R);
    const int Mtop = (Rint < GEMM_ROW_TILE * num_sms()) ? Rint : GEMM_ROW_TILE * num_sms();
    for (int i = 0; i <= N; ++i) {
        for (int M = GEMM_ROW_TILE; ; M += GEMM_ROW_TILE) {
            const size_t b = ctcb_gemm_workspace_bytes(M <= Mtop ? M : Rint, sizes[i + 1], sizes[i]);
            if (b > g) g = b;
            if (M > Mtop) break;
        }
    }
    const WsLayout w = ws_layout(c);
    const size_t train_area = w.gemm2 - w.gemm;
    f.gemm = take(g < train_area ? g : train_area);
    f.gemm_bytes = off - f.gemm;
    f.counters = take(sizeof(unsigned int) * 1024);
    f.sweep_bytes = eff_tl(c) ? sweep_tc_workspace_bytes(H, c->maxB) : 0;     // as in ws_layout: same sweep plan
    f.sweep = take(f.sweep_bytes);
    f.total = off;
    return f;
}
}  // namespace

extern "C" size_t ctcb_brnn_workspace_bytes(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    return ws_layout(cfg).total;
}

extern "C" size_t ctcb_brnn_forward_workspace_bytes(const ctcb_brnn_config *cfg, size_t *error_flag_offset) {
    if (!valid_cfg(cfg)) return 0;
    const FwdLayout f = fwd_layout(cfg);
    if (error_flag_offset) *error_flag_offset = f.counters;
    return f.total;
}

extern "C" size_t ctcb_brnn_error_flag_offset(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    return ws_layout(cfg).counters;
}

extern "C" int ctcb_brnn_create(const ctcb_brnn_config *cfg, ctcb_brnn **out) {
    if (cfg && cfg->maxLabels > CTCB_CTC_MAX_LABELS)
        return set_error(CTCB_EINVAL, "ctcb_brnn_create: maxLabels %d exceeds the CTC kernel's limit of %d labels per utterance",
                         cfg->maxLabels, CTCB_CTC_MAX_LABELS);
    if (cfg && cfg->numTemporal > 1 && !valid_cfg(cfg))
        return set_error(CTCB_EINVAL, "ctcb_brnn_create: a block of %d temporal layers from layer %d does not fit in "
                         "hidden layers 1..%d", cfg->numTemporal, cfg->temporalLayer, cfg->numLayers);
    if (!valid_cfg(cfg) || !out) return set_error(CTCB_EINVAL, "ctcb_brnn_create: bad config");
    ctcb_brnn *h = new (std::nothrow) ctcb_brnn;
    if (!h) return set_error(CTCB_ENOMEM, "ctcb_brnn_create: out of host memory");
    h->cfg = *cfg;
    if (h->cfg.maxAct <= 0.f) h->cfg.maxAct = 20.0f;   // brnnet.py:32
    h->nlayers = cfg->numLayers + 1;
    h->tl = eff_tl(cfg);
    h->nt = eff_nt(cfg);
    layer_sizes(cfg, h->sizes);
    h->side = nullptr;
    h->side_ready = false;
    h->defer_l2 = false;
    h->comm = nullptr;
    h->fwd_ready = false;
    *out = h;
    return CTCB_OK;
}

extern "C" void ctcb_brnn_destroy(ctcb_brnn *h) {
    if (h && h->side_ready) {
        cudaStreamDestroy(h->side);
        for (int i = 0; i < 66; ++i) cudaEventDestroy(h->ev_delta[i]);
        cudaEventDestroy(h->ev_side);
        for (int p = 0; p < 2; ++p) cudaEventDestroy(h->ev_pair[p]);
    }
    delete h;
}

static int ensure_side_stream(ctcb_brnn *h) {
    if (h->side_ready) return CTCB_OK;
    CTCB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
    for (int i = 0; i < 66; ++i) CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_delta[i], cudaEventDisableTiming));
    CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_side, cudaEventDisableTiming));
    for (int p = 0; p < 2; ++p) CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_pair[p], cudaEventDisableTiming));
    h->side_ready = true;
    return CTCB_OK;
}

#define TRY(expr)                    \
    do {                             \
        int _rc = (expr);            \
        if (_rc != CTCB_OK) return _rc; \
    } while (0)

extern "C" int ctcb_brnn_sweep_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, const float *pre,
                                   const float *Wf, const float *Wb, float *outF, float *outB, const float *actF,
                                   const float *actB, float maxAct, void *scratch, size_t scratch_bytes, void *stream) {
    if (!T_per_utt || !pre || !Wf || !outF || !scratch || (mode == 1 && !actF) ||
        (Wb && (!outB || (mode == 1 && !actB))))
        return set_error(CTCB_EINVAL, "ctcb_brnn_sweep_f32: null pointer argument");
    if (T <= 0 || B <= 0 || H <= 0 || (mode != 0 && mode != 1))
        return set_error(CTCB_EINVAL, "ctcb_brnn_sweep_f32: bad sizes");
    CTCB_CUDA_CHECK(cudaMemsetAsync(scratch, 0, 16 * sizeof(unsigned int), (cudaStream_t)stream));   // error flag
    if (scratch_bytes < 4096) return set_error(CTCB_ENOMEM, "ctcb_brnn_sweep_f32: scratch %zu < 4096 bytes", scratch_bytes);
    return run_sweep(mode, T, B, H, T_per_utt, pre, Wf, Wb, outF, outB, actF, actB, maxAct,
                     (unsigned int *)scratch, (char *)scratch + 4096, scratch_bytes - 4096, (cudaStream_t)stream);
}

// The part of the flat gradient that was NOT summed early on the side stream, plus the statistics tail, in one grouped
// NCCL launch: with an early bucket [off(2 tl), end of layer N+1), tl the lowest temporal layer, that is everything
// before it and everything behind it (the recurrent matrices of every temporal layer among them).
static int brnn_reduce_rest(ctcb_brnn *h, float *grads, float *stats, bool early_bucket, cudaStream_t st) {
    const ctcb_brnn_config &c = h->cfg;
    const int64_t P = ctcb_brnn_param_count(&c);
    float *ptrs[3];
    int64_t cnt[3];
    int k = 0;
    int64_t lo = P, hi = P;      // [lo, hi) was reduced early
    if (early_bucket) {
        int64_t o; int32_t r, cc;
        ctcb_brnn_tensor_info(&c, 2 * h->tl, &lo, nullptr, nullptr);
        ctcb_brnn_tensor_info(&c, 2 * c.numLayers + 1, &o, &r, &cc);
        hi = o + (int64_t)r * cc;
    }
    ptrs[k] = grads; cnt[k] = lo; ++k;
    const bool tail_adjacent = (stats == grads + P);
    ptrs[k] = grads + hi; cnt[k] = P - hi + (stats && tail_adjacent ? 4 : 0); ++k;
    if (stats && !tail_adjacent) { ptrs[k] = stats; cnt[k] = 4; ++k; }
    return comm_allreduce_ranges(h->comm, ptrs, cnt, k, st);
}

// Where the forward half reads and writes: X[i] (1..N+1) the output of affine map i (pre-activation, then For+Back,
// at a temporal layer; the logits at N+1), the two sweep outputs of each temporal layer j (one pair shared by all
// layers in the forward-only layout), the split-K area, the sweep counters and scratch.
struct FwdBufs {
    float *X[66];
    float *For[64], *Back[64];
    void *gemm;
    size_t gemm_bytes;
    unsigned int *counters;
    void *sweep;
    size_t sweep_bytes;
};

// brnnet.py:136-173: the affine maps with bias(+ReLU) fused, the two-direction sweep and For+Back at each temporal
// layer, the softmax into probs_out when given.  Clears the sweep error flag first.
static int brnn_forward(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt, int B, int Tmax,
                        const float *params, float *probs_out, const FwdBufs &m, cudaStream_t st) {
    const ctcb_brnn_config &c = h->cfg;
    const int N = c.numLayers, H = c.layerSize, K = c.outputDim, tl = h->tl, nt = h->nt;
    const int *sz = h->sizes;
    const int64_t R = (int64_t)Tmax * B;
    auto P = [&](int idx) -> const float * {
        int64_t off; ctcb_brnn_tensor_info(&c, idx, &off, nullptr, nullptr); return params + off;
    };
    const bool uni = (c.unidirectional != 0);
    auto temporal = [&](int i) { return nt > 0 && i >= tl && i < tl + nt; };
    // the uni-directional temporal layer's output IS the forward sweep (rnnet.py:112-116)
    auto Act = [&](int i) -> const float * { return (uni && temporal(i)) ? m.For[i - tl] : m.X[i]; };
    // the sweep kernels' error flag (word 0) is cleared once per call, so a forward-sweep timeout survives the BPTT sweep
    CTCB_CUDA_CHECK(cudaMemsetAsync(m.counters, 0, 16 * sizeof(unsigned int), st));
    for (int i = 1; i <= N + 1; ++i) {
        const float *in = (i == 1) ? feats : Act(i - 1);
        const int relu = (i <= N && !temporal(i)) ? 1 : 0;
        {
        ProfScope ps("gemm_fwd", st);
        TRY(ctcb_gemm_f32(0, 1, (int)R, sz[i], sz[i - 1], 1.f, in, sz[i - 1], P(2 * (i - 1)), sz[i - 1], 0.f,
                          m.X[i], sz[i], P(2 * (i - 1) + 1), relu, nullptr, m.gemm, m.gemm_bytes, st));
        }
        if (temporal(i)) {
            const int j = i - tl, iWtf = rec_index(&c, j);
            {
            ProfScope ps("sweep_fwd", st);
            TRY(run_sweep(0, Tmax, B, H, T_per_utt, m.X[i], P(iWtf), uni ? nullptr : P(iWtf + 2), m.For[j], m.Back[j],
                          nullptr, nullptr, c.maxAct, m.counters, m.sweep, m.sweep_bytes, st));
            }
            if (!uni) {     // over the pre-activation, which nothing reads after the sweep
                ProfScope ps("elementwise", st);
                TRY(run_add2(m.For[j], m.Back[j], m.X[i], R * H, st));     // brnnet.py:153
            }
        }
    }
    if (probs_out) {
        const int wpb = 8;
        softmax_rows_kernel<<<(unsigned)((R + wpb - 1) / wpb), wpb * 32, 0, st>>>(m.X[N + 1], probs_out, R, K);
        CTCB_LAUNCH_CHECK();
    }
    return CTCB_OK;
}

// One micro-batch of a step whose gradient is the sum over several calls (include/ctcb200.h): without
// CTCB_PART_FIRST every gradient tensor and the statistics tail are added into, with it overwritten; only the
// CTCB_PART_LAST call exchanges over the ranks and adds the L2 term, so each happens once per step.
// ctcb_brnn_cost_and_grad is this with both flags.
extern "C" int ctcb_brnn_cost_and_grad_part(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt,
                                            const int32_t *labels, const int32_t *label_off, int B, int Tmax,
                                            const float *params, float *grads, float *cost_out, int32_t *skip_out,
                                            float *regcost_out, float *probs_out, float *stats_out, int flags,
                                            void *workspace, size_t ws_bytes, void *stream) {
    if (!h || !feats || !T_per_utt || !params)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: null pointer argument");
    if (flags & ~(CTCB_PART_FIRST | CTCB_PART_LAST))
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad_part: unknown flags 0x%x", flags);
    const bool first = (flags & CTCB_PART_FIRST) != 0, last = (flags & CTCB_PART_LAST) != 0;
    const float beta_g = first ? 0.f : 1.f;      // weight-gradient contractions: C = dW (+ C)
    const ctcb_brnn_config &c = h->cfg;
    if (B <= 0 || B > c.maxB || Tmax <= 0 || Tmax > c.maxT)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: batch %d x %d frames exceeds the configured %d x %d",
                         B, Tmax, c.maxB, c.maxT);
    const bool train = (grads != nullptr);
    if (train && (!labels || !label_off || !cost_out || !skip_out))
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: training mode needs labels and cost/skip outputs");
    if (!train && !probs_out)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: forward-only mode needs probs_out");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    const int N = c.numLayers, H = c.layerSize, K = c.outputDim, tl = h->tl;
    const int *sz = h->sizes;
    const int64_t R = (int64_t)Tmax * B;
    if (R > 0x7fffffff) return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: T*B too large");
    FwdBufs m{};
    if (!train) {     // the forward layout whatever the size given: the same kernels and plans as a training call
        if (!h->fwd_ready) {
            h->fwd = fwd_layout(&c);
            h->fwd_ready = true;
        }
        const FwdLayout &f = h->fwd;
        if (!workspace || ws_bytes < f.total)
            return set_error(CTCB_ENOMEM, "ctcb_brnn_cost_and_grad: workspace %zu < %zu bytes", ws_bytes, f.total);
        for (int i = 1; i <= N + 1; ++i) m.X[i] = (float *)(ws + f.slab[i % 2]);
        for (int j = 0; j < h->nt; ++j) {     // one pair for every temporal layer: each sweep runs after the last read
            m.For[j] = f.For ? (float *)(ws + f.For) : nullptr;   // offset 0 is slab 0: For / Back were not laid out
            m.Back[j] = f.Back ? (float *)(ws + f.Back) : nullptr;
        }
        m.gemm = ws + f.gemm;
        m.gemm_bytes = f.gemm_bytes;
        m.counters = (unsigned int *)(ws + f.counters);
        m.sweep = ws + f.sweep;
        m.sweep_bytes = f.sweep_bytes;
        return brnn_forward(h, feats, T_per_utt, B, Tmax, params, probs_out, m, st);
    }
    const WsLayout w = ws_layout(&c);
    if (!workspace || ws_bytes < w.total)
        return set_error(CTCB_ENOMEM, "ctcb_brnn_cost_and_grad: workspace %zu < %zu bytes", ws_bytes, w.total);
    auto Xbuf = [&](int i) -> float * { return (float *)(ws + w.X[i]); };
    auto P = [&](int idx) -> const float * {
        int64_t off; ctcb_brnn_tensor_info(&c, idx, &off, nullptr, nullptr); return params + off;
    };
    auto G = [&](int idx) -> float * {
        int64_t off; ctcb_brnn_tensor_info(&c, idx, &off, nullptr, nullptr); return grads + off;
    };
    // For_j / Back_j of temporal layer j; the dFor / dBack pair of layer j is pair j % 2
    float *ForJ[64], *BackJ[64];
    for (int j = 0; j < h->nt; ++j) {
        ForJ[j] = (float *)(ws + w.ForJ[j]);
        BackJ[j] = (float *)(ws + w.BackJ[j]);      // unused (offset 0) for the uni-directional layers above the first
    }
    float *dF[2] = {(float *)(ws + w.dFor), (float *)(ws + w.dFor2)};
    float *dB[2] = {(float *)(ws + w.dBack), (float *)(ws + w.dBack2)};
    void *gws = ws + w.gemm;
    const size_t gws_bytes = w.gemm2 - w.gemm;
    unsigned int *counters = (unsigned int *)(ws + w.counters);
    const int nt = h->nt;
    const bool uni = (c.unidirectional != 0);
    auto temporal = [&](int i) { return nt > 0 && i >= tl && i < tl + nt; };
    // activations of layer i as the next layer (and the weight gradients) see them: a uni-directional temporal
    // layer's output IS its forward sweep (rnnet.py:112-116), a bi-directional one's is For + Back
    auto Act = [&](int i) -> float * { return (uni && temporal(i)) ? ForJ[i - tl] : Xbuf(i); };

    // ---------------------------------------------------------------- forward (brnnet.py:136-157)
    for (int i = 1; i <= N + 1; ++i) m.X[i] = Xbuf(i);
    for (int j = 0; j < nt; ++j) {
        m.For[j] = ForJ[j];
        m.Back[j] = BackJ[j];
    }
    m.gemm = gws;
    m.gemm_bytes = gws_bytes;
    m.counters = counters;
    m.sweep = ws + w.sweep;
    m.sweep_bytes = w.sweep_bytes;
    TRY(brnn_forward(h, feats, T_per_utt, B, Tmax, params, probs_out, m, st));
    float *logits = Xbuf(N + 1);

    // ---------------------------------------------------------------- CTC (brnnet.py:161-175)
    auto dbuf = [&](int j) -> float * { return (float *)(ws + w.D[j]); };
    {
    ProfScope ps("ctc", st);
    TRY(ctcb_ctc_loss_grad_f32(logits, 0, (int64_t)K, (int64_t)B * K, labels, label_off, T_per_utt, B, Tmax, K,
                               c.maxLabels, 0, dbuf(N + 1), cost_out, skip_out, ws + w.ctc, w.gemm - w.ctc, st));
    }

    // ---------------------------------------------------------------- backward (brnnet.py:188-243)
    // Per temporal layer from the top: the delta GEMM without a mask, the BPTT sweep into pair j % 2, the recurrent
    // weight-gradient pair on the side stream, add2.  Layer j - 2 writes the pair layer j used: its sweep waits for
    // ev_pair, recorded on the side stream behind the last read of that pair (the recurrent weight gradients; for a
    // uni-directional layer the weight gradient of the map above, whose delta the pair is).
    const bool overlap = (tl > 0);     // layers i >= tl: dW/db on the side stream, delta chain + BPTT on the main one
    const bool dp = (h->comm != nullptr) && comm_world(h->comm) > 1;
    if (overlap) TRY(ensure_side_stream(h));
    void *gws2 = ws + w.gemm2;
    const size_t gws2_bytes = w.colsum - w.gemm2;
    for (int i = N; i >= 0; --i) {
        const float *Xi = (i == 0) ? feats : Act(i);
        const int n_out = sz[i + 1], n_in = sz[i];
        // rnnet.py:162-177: the BPTT result of a uni-directional layer is the delta
        float *dcur = (uni && temporal(i + 1)) ? dF[(i + 1 - tl) % 2] : dbuf(i + 1);
        const bool on_side = overlap && i >= tl;
        cudaStream_t sw = on_side ? h->side : st;
        if (on_side) {     // dcur is complete on the main stream here
            CTCB_CUDA_CHECK(cudaEventRecord(h->ev_delta[i], st));
            CTCB_CUDA_CHECK(cudaStreamWaitEvent(h->side, h->ev_delta[i], 0));
        }
        // dW = delta^T . X_i   (brnnet.py:196)
        {
        ProfScope ps("gemm_dw", sw);
        TRY(ctcb_gemm_f32(1, 0, n_out, n_in, (int)R, 1.f, dcur, n_out, Xi, n_in, beta_g, G(2 * i), n_in, nullptr, 0,
                          nullptr, on_side ? gws2 : gws, on_side ? gws2_bytes : gws_bytes, sw));
        }
        // db = row sums of delta   (brnnet.py:200)
        {
            ProfScope ps("colsum", sw);
            float *part = (float *)(ws + (on_side ? w.colsum2 : w.colsum));
            int nblk;
            if (n_out % 4 == 0 && (((uintptr_t)dcur) & 15) == 0) {
                const int n4 = n_out / 4;
                const int bx = n4 >= 256 ? 256 : (n4 + 31) / 32 * 32;
                const int ncb = (n4 + bx - 1) / bx;
                int64_t rpb = R / (2 * num_sms() / ncb > 0 ? 2 * num_sms() / ncb : 1);     // ~2 blocks per SM
                if (rpb < CS_ROWS_MIN) rpb = CS_ROWS_MIN;
                if (rpb > CS_ROWS) rpb = CS_ROWS;
                nblk = (int)((R + rpb - 1) / rpb);
                colsum_stage1_wide<<<dim3(ncb, nblk), bx, 0, sw>>>((const float4 *)dcur, R, n4, (int)rpb, (float4 *)part);
            } else {
                nblk = (int)((R + CS_ROWS - 1) / CS_ROWS);
                colsum_stage1<<<dim3((n_out + 31) / 32, nblk), dim3(32, 8), 0, sw>>>(dcur, R, n_out, part);
            }
            CTCB_LAUNCH_CHECK();
            if (first) colsum_stage2<false><<<(n_out + 127) / 128, 128, 0, sw>>>(part, nblk, n_out, G(2 * i + 1));
            else colsum_stage2<true><<<(n_out + 127) / 128, 128, 0, sw>>>(part, nblk, n_out, G(2 * i + 1));
            CTCB_LAUNCH_CHECK();
        }
        if (uni && temporal(i + 1) && i + 1 - tl >= 2)     // the last read of the pair of uni-directional layer i + 1
            CTCB_CUDA_CHECK(cudaEventRecord(h->ev_pair[(i + 1 - tl) % 2], h->side));
        if (dp && last && on_side && i == tl) {
            // every gradient tensor of the layers >= tl is now queued on the side stream: sum that contiguous range over
            // the ranks there, next to the BPTT sweep on the main stream
            float *pa = G(2 * tl);
            const int64_t na = (G(2 * N + 1) + sz[N + 1]) - pa;
            TRY(comm_allreduce_ranges(h->comm, &pa, &na, 1, h->side));
        }
        if (i > 0) {
            float *doth = dbuf(i);
            // delta <- delta . W, with the ReLU mask sign(hActs[i]) fused (brnnet.py:203-204,235-237)
            const float *mask = temporal(i) ? nullptr : Xi;
            {
            ProfScope ps("gemm_delta", st);
            TRY(ctcb_gemm_f32(0, 0, (int)R, n_in, n_out, 1.f, dcur, n_out, P(2 * i), n_in, 0.f, doth, n_in,
                              nullptr, 0, mask, gws, gws_bytes, st));
            }
            if (temporal(i)) {   // brnnet.py:207-233
                const int j = i - tl, p = j % 2, iWtf = rec_index(&c, j), iWtb = iWtf + 2;
                float *dFor = dF[p], *dBack = dB[p], *For = ForJ[j], *Back = BackJ[j];
                if (j + 2 < nt)      // layer j + 2 used this pair
                    CTCB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_pair[p], 0));
                {
                ProfScope ps("sweep_bptt", st);
                TRY(run_sweep(1, Tmax, B, H, T_per_utt, doth, P(iWtf), uni ? nullptr : P(iWtb), dFor, dBack, For, Back,
                              c.maxAct, counters, ws + w.sweep, w.sweep_bytes, st));
                }
                // recurrent weight gradients (brnnet.py:227-230): independent of the rest of the backward pass,
                // so they go to the side stream as well
                CTCB_CUDA_CHECK(cudaEventRecord(h->ev_delta[65], st));
                CTCB_CUDA_CHECK(cudaStreamWaitEvent(h->side, h->ev_delta[65], 0));
                {
                ProfScope ps("gemm_dw_rec", h->side);
                if (Tmax > 1) {
                    const int64_t Rm = R - B;
                    if (uni)
                        TRY(ctcb_gemm_f32(1, 0, H, H, (int)Rm, 1.f, dFor + (int64_t)B * H, H, For, H, beta_g, G(iWtf), H,
                                          nullptr, 0, nullptr, gws2, gws2_bytes, h->side));
                    else     // both directions in one launch
                        TRY(ctcb_gemm_pair_f32(1, 0, H, H, (int)Rm, 1.f, dFor + (int64_t)B * H, dBack, H, For,
                                               Back + (int64_t)B * H, H, beta_g, G(iWtf), G(iWtb), H, gws2, gws2_bytes,
                                               h->side));
                } else if (first) {     // one frame: no recurrence, nothing to add to earlier micro-batches
                    CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtf), 0, sizeof(float) * H * H, h->side));
                    if (!uni) CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtb), 0, sizeof(float) * H * H, h->side));
                }
                }
                if (!uni) {
                    if (j >= 2) CTCB_CUDA_CHECK(cudaEventRecord(h->ev_pair[p], h->side));
                    TRY(run_add2(dFor, dBack, doth, R * H, st));
                }
            }
        }
    }
    if (overlap) {     // join: every gradient tensor is complete on the caller's stream from here on
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_side, h->side));
        CTCB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_side, 0));
    }
    for (int j = 0; j < nt; ++j) {   // the `dummy` biases never receive gradient
        const int iWtf = rec_index(&c, j);
        CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtf + 1), 0, sizeof(float), st));
        if (!uni) CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtf + 3), 0, sizeof(float), st));
    }

    if (stats_out) {     // after both sweeps, so that the tail carries the error flag of either
        if (first) batch_stats_kernel<false><<<1, 32, 0, st>>>(cost_out, skip_out, B, stats_out, counters);
        else batch_stats_kernel<true><<<1, 32, 0, st>>>(cost_out, skip_out, B, stats_out, counters);
        CTCB_LAUNCH_CHECK();
    }
    // an earlier micro-batch of the step: the exchange and the L2 term wait for the sum of all of them
    if (!last) return CTCB_OK;

    if (dp) TRY(brnn_reduce_rest(h, grads, stats_out, overlap, st));

    // ---------------------------------------------------------------- L2 (brnnet.py:177-183,197-198,244-247)
    if (regcost_out) {
        set_scalar_kernel<<<1, 1, 0, st>>>(regcost_out, 0.f);
        CTCB_LAUNCH_CHECK();
    }
    if (c.reg > 0.f) {
        const int nt = ctcb_brnn_num_tensors(&c);
        for (int idx = 0; idx < nt; idx += 2) {
            int64_t off; int32_t r, cc;
            ctcb_brnn_tensor_info(&c, idx, &off, &r, &cc);
            const int64_t n = (int64_t)r * cc;
            if (!h->defer_l2) TRY(ctcb_axpy_f32(grads + off, params + off, c.reg, n, st));
            if (regcost_out) TRY(run_sumsq(params + off, n, regcost_out, 0.5f * c.reg, 1, ws + w.scratch, st));
        }
    }
    return CTCB_OK;
}

extern "C" int ctcb_brnn_cost_and_grad(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt,
                                       const int32_t *labels, const int32_t *label_off, int B, int Tmax,
                                       const float *params, float *grads, float *cost_out, int32_t *skip_out,
                                       float *regcost_out, float *probs_out, float *stats_out, void *workspace,
                                       size_t ws_bytes, void *stream) {
    return ctcb_brnn_cost_and_grad_part(h, feats, T_per_utt, labels, label_off, B, Tmax, params, grads, cost_out,
                                        skip_out, regcost_out, probs_out, stats_out,
                                        CTCB_PART_FIRST | CTCB_PART_LAST, workspace, ws_bytes, stream);
}

extern "C" int ctcb_brnn_set_deferred_l2(ctcb_brnn *h, int deferred) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_deferred_l2: null handle");
    h->defer_l2 = (deferred != 0);
    return CTCB_OK;
}

extern "C" int ctcb_brnn_apply_l2_f32(ctcb_brnn *h, const float *params, float *grads, void *stream) {
    if (!h || !params || !grads) return set_error(CTCB_EINVAL, "ctcb_brnn_apply_l2_f32: null pointer argument");
    const ctcb_brnn_config &c = h->cfg;
    if (c.reg <= 0.f) return CTCB_OK;
    const int nt = ctcb_brnn_num_tensors(&c);
    for (int idx = 0; idx < nt; idx += 2) {     // weight matrices only, as brnnet.py:197-198,244-247
        int64_t off; int32_t r, cc;
        ctcb_brnn_tensor_info(&c, idx, &off, &r, &cc);
        TRY(ctcb_axpy_f32(grads + off, params + off, c.reg, (int64_t)r * cc, stream));
    }
    return CTCB_OK;
}

extern "C" int ctcb_brnn_set_comm(ctcb_brnn *h, ctcb_comm *comm) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_comm: null handle");
    h->comm = comm;
    return CTCB_OK;
}

// The exchange half of a data-parallel step for a rank that had NO utterance this step: `grads` (zero-filled by the
// caller, statistics tail included) goes through the same sequence of collectives as ctcb_brnn_cost_and_grad issues.
extern "C" int ctcb_brnn_exchange_only(ctcb_brnn *h, const float *params, float *grads, float *stats_out, void *stream) {
    if (!h || !params || !grads) return set_error(CTCB_EINVAL, "ctcb_brnn_exchange_only: null pointer argument");
    if (!h->comm || comm_world(h->comm) <= 1) return CTCB_OK;
    const ctcb_brnn_config &c = h->cfg;
    cudaStream_t st = (cudaStream_t)stream;
    const bool early = (h->tl > 0);
    if (early) {
        int64_t lo, o; int32_t r, cc;
        ctcb_brnn_tensor_info(&c, 2 * h->tl, &lo, nullptr, nullptr);
        ctcb_brnn_tensor_info(&c, 2 * c.numLayers + 1, &o, &r, &cc);
        float *pa = grads + lo;
        const int64_t na = o + (int64_t)r * cc - lo;
        TRY(comm_allreduce_ranges(h->comm, &pa, &na, 1, st));
    }
    TRY(brnn_reduce_rest(h, grads, stats_out, early, st));
    if (c.reg > 0.f && !h->defer_l2) return ctcb_brnn_apply_l2_f32(h, params, grads, stream);
    return CTCB_OK;
}

extern "C" size_t ctcb_brnn_sweep_workspace_bytes(int H, int B) { return 4096 + ctcb::sweep_tc_workspace_bytes(H, B); }

// Test / diagnostic hook: where, inside the workspace, the activations of the LAST ctcb_brnn_cost_and_grad call lie
// (time-major [Tmax][B][n] with that call's B and Tmax).  what = 0: output of affine map `layer` (1..numLayers+1; the
// temporal layer's entry holds For + Back, the last one the logits), 1: For, 2: Back (temporal layer only; with
// several, `layer` says which).
extern "C" int ctcb_brnn_activation_offset(const ctcb_brnn_config *cfg, int what, int layer, size_t *offset, int32_t *width) {
    if (!valid_cfg(cfg) || !offset) return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: bad arguments");
    const WsLayout w = ws_layout(cfg);
    int sizes[66];
    layer_sizes(cfg, sizes);
    if (what == 0) {
        if (layer < 1 || layer > cfg->numLayers + 1) return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d", layer);
        *offset = w.X[layer];
        if (width) *width = sizes[layer];
        return CTCB_OK;
    }
    const int nt = eff_nt(cfg);
    if ((what == 1 || what == 2) && nt == 1) {     // one temporal layer: `layer` is ignored
        *offset = (what == 1) ? w.For : w.Back;
        if (width) *width = cfg->layerSize;
        return CTCB_OK;
    }
    if ((what == 1 || (what == 2 && !cfg->unidirectional)) && nt > 1) {
        const int j = layer - eff_tl(cfg);
        if (j < 0 || j >= nt)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d is not one of the temporal layers %d..%d",
                             layer, eff_tl(cfg), eff_tl(cfg) + nt - 1);
        *offset = (what == 1) ? w.ForJ[j] : w.BackJ[j];
        if (width) *width = cfg->layerSize;
        return CTCB_OK;
    }
    return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: nothing of kind %d in this net", what);
}
