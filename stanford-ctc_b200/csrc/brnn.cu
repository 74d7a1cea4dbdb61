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
#include <cmath>
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
int run_dropout(float *X, int64_t R, int B, int H, int layer, uint64_t seed, const int64_t *step, int64_t first,
                int64_t stride, uint32_t thr, float scale, cudaStream_t st);
const char *input_mask_layout_error(int D, int nu, char (&buf)[192]);
const char *input_mask_policy_error(int nu, int mF, int F, int mT, int Tw, double p, char (&buf)[192]);
int run_input_mask(const float *x, const int32_t *lens, int B, int Tmax, int D, int nu, int mF, int F, int mT, int Tw,
                   double p, uint64_t seed, const int64_t *step, int64_t first, int64_t stride, float *y,
                   cudaStream_t st);
int run_weight_noise(const float *w, float *y, int64_t n, const int64_t *lo, const int64_t *hi, int nr, float sigma,
                     uint64_t seed, const int64_t *step, cudaStream_t st);
size_t lstm_carry_bytes(int H, int B);
int run_lstm_sweep(int mode, int T, int B, int H, const int32_t *Tlen, float *gates, const float *Uf, const float *Ub,
                   const float *Pf, const float *Pb, float *hF, float *hB, float *cF, float *cB, const float *dh,
                   float *dz, unsigned int *counters, float *dc, const LstmZoneout *zo, cudaStream_t st);
int lstm_check(int H, int B, int ndir, bool peep, bool zo);
int sweep_check(int H, int B, int ndir);
size_t lstm_peephole_grad_bytes(int64_t R, int H, int ndir);
int run_lstm_peephole_grad(int T, int B, int H, const float *dz, const float *cF, const float *cB, float *dPf,
                           float *dPb, bool accumulate, float *partial, cudaStream_t st);
size_t layernorm_workspace_bytes(int64_t R, int H);
int run_layernorm_forward(const float *z, float *y, float *mu, float *rstd, const float *gamma, const float *beta,
                          int64_t R, int H, cudaStream_t st);
int run_layernorm_backward(float *d, const float *z, const float *mu, const float *rstd, const float *gamma,
                           float *dgamma, float *dbeta, int64_t R, int H, bool accumulate, float *partial,
                           cudaStream_t st);
int64_t subsampled_frames(int T, int k);
int run_frame_stack(const float *x, const int32_t *Tlen, int Tmax, int B, int n, int k, float *s_out, int32_t *lens_out,
                    cudaStream_t st);
int run_frame_unstack(const float *ds, const int32_t *Tlen, int Tmax, int B, int n, int k, float *d_out, cudaStream_t st);

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

// out = p (dp - sum_k p_k dp_k) + add per row: the backward of the row softmax (self-conditioned CTC's dA); one warp per
// row.  out may alias dp: each lane reads its elements of dp before the warp sum and writes only those after it.
__global__ void softmax_rows_backward_kernel(const float *__restrict__ p, const float *dp, const float *__restrict__ add,
                                             float *out, int64_t R, int K) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= R) return;
    const float *pr = p + row * K, *dr = dp + row * K;
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s = fmaf(pr[k], dr[k], s);
    s = warp_sum(s);
    for (int k = lane; k < K; k += 32) {
        const float v = pr[k] * (dr[k] - s);
        out[row * K + k] = add ? v + add[row * K + k] : v;
    }
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

// the intermediate CTC's pair of the statistics tail: stats[0] += the sum of its nll over the utterances it kept,
// stats[1] += the number it skipped (= with ACC false); one warp
template <bool ACC>
__global__ void inter_stats_kernel(const float *__restrict__ cost, const int32_t *__restrict__ skip, int B, float *stats) {
    float cs = 0.f, ns = 0.f;
    for (int u = threadIdx.x; u < B; u += 32) {
        if (skip[u]) ns += 1.f;
        else cs += cost[u];
    }
    cs = warp_sum(cs); ns = warp_sum(ns);
    if (threadIdx.x == 0) {
        if (ACC) { cs += stats[0]; ns += stats[1]; }
        stats[0] = cs; stats[1] = ns;
    }
}

// x[0..n) *= s in place (the intermediate loss's weight on its CTC gradient)
__global__ void scale_kernel(float *__restrict__ x, int64_t n, float s) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        x[i] *= s;
}

// The stage-1 grid of run_colsum: the wide kernel (n % 4 == 0 and a 16-byte aligned delta) over ncb column blocks of
// bx threads and row blocks of rpb rows, or the narrow one over ncb blocks of 32 columns and row blocks of CS_ROWS rows
struct ColsumPlan {
    bool wide;
    int ncb, bx;
    int64_t rpb;
    int nblk;
};
ColsumPlan colsum_plan(const float *delta, int64_t R, int n) {
    ColsumPlan p{};
    p.wide = n % 4 == 0 && (((uintptr_t)delta) & 15) == 0;
    if (p.wide) {
        const int n4 = n / 4;
        p.bx = n4 >= 256 ? 256 : (n4 + 31) / 32 * 32;
        p.ncb = (n4 + p.bx - 1) / p.bx;
        p.rpb = R / (2 * num_sms() / p.ncb > 0 ? 2 * num_sms() / p.ncb : 1);     // ~2 blocks per SM
        if (p.rpb < CS_ROWS_MIN) p.rpb = CS_ROWS_MIN;
        if (p.rpb > CS_ROWS) p.rpb = CS_ROWS;
    } else {
        p.bx = 32;
        p.ncb = (n + 31) / 32;
        p.rpb = CS_ROWS;
    }
    p.nblk = (int)((R + p.rpb - 1) / p.rpb);
    return p;
}

// both stages of the column sums of the row-major R x n matrix `delta` into out[n]; `partial` holds one row of n floats
// per CS_ROWS_MIN rows of R
int run_colsum(const float *delta, int64_t R, int n, float *partial, float *out, bool accumulate, cudaStream_t st) {
    const ColsumPlan p = colsum_plan(delta, R, n);
    if (p.wide)
        colsum_stage1_wide<<<dim3(p.ncb, p.nblk), p.bx, 0, st>>>((const float4 *)delta, R, n / 4, (int)p.rpb,
                                                                (float4 *)partial);
    else
        colsum_stage1<<<dim3(p.ncb, p.nblk), dim3(32, 8), 0, st>>>(delta, R, n, partial);
    CTCB_LAUNCH_CHECK();
    if (!accumulate) colsum_stage2<false><<<(n + 127) / 128, 128, 0, st>>>(partial, p.nblk, n, out);
    else colsum_stage2<true><<<(n + 127) / 128, 128, 0, st>>>(partial, p.nblk, n, out);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

// the row softmax of the forward-only output: one warp per row, 8 rows per block
int run_softmax_rows(const float *x, float *p, int64_t R, int K, cudaStream_t st) {
    const int wpb = 8;
    softmax_rows_kernel<<<(unsigned)((R + wpb - 1) / wpb), wpb * 32, 0, st>>>(x, p, R, K);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

// its backward, in the same grid
int run_softmax_rows_backward(const float *p, const float *dp, const float *add, float *out, int64_t R, int K,
                              cudaStream_t st) {
    const int wpb = 8;
    softmax_rows_backward_kernel<<<(unsigned)((R + wpb - 1) / wpb), wpb * 32, 0, st>>>(p, dp, add, out, R, K);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

int run_batch_stats(const float *cost, const int32_t *skip, int B, float *stats, const unsigned int *errflag,
                    bool accumulate, cudaStream_t st) {
    if (!accumulate) batch_stats_kernel<false><<<1, 32, 0, st>>>(cost, skip, B, stats, errflag);
    else batch_stats_kernel<true><<<1, 32, 0, st>>>(cost, skip, B, stats, errflag);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

int run_inter_stats(const float *cost, const int32_t *skip, int B, float *stats, bool accumulate, cudaStream_t st) {
    if (!accumulate) inter_stats_kernel<false><<<1, 32, 0, st>>>(cost, skip, B, stats);
    else inter_stats_kernel<true><<<1, 32, 0, st>>>(cost, skip, B, stats);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

int run_scale(float *x, int64_t n, float s, cudaStream_t st) {
    const int64_t blocks = (n + 255) / 256;
    scale_kernel<<<(unsigned)(blocks < 4 * num_sms() ? blocks : 4 * num_sms()), 256, 0, st>>>(x, n, s);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}

}  // namespace ctcb

using namespace ctcb;

#define TRY(expr)                    \
    do {                             \
        int _rc = (expr);            \
        if (_rc != CTCB_OK) return _rc; \
    } while (0)

// ---- the config: validity, layer sizes, the flat parameter vector ------------------------------
// Why a config cannot be used, worded for the caller of ctcb_brnn_create (into `buf` where it has numbers), or null.
static const char *cfg_error(const ctcb_brnn_config *c, char (&buf)[192]) {
    auto say = [&buf](const char *fmt, auto... args) -> const char * {
        snprintf(buf, sizeof(buf), fmt, args...);
        return buf;
    };
    if (!c) return "bad config";
    if (c->maxLabels > CTCB_CTC_MAX_LABELS)     // the CTC kernel's register-resident trellis (ctc.cu)
        return say("maxLabels %d exceeds the CTC kernel's limit of %d labels per utterance", c->maxLabels,
                   CTCB_CTC_MAX_LABELS);
    if ((int64_t)c->maxT * c->maxB > GEMM_MAX_M)     // the forward and delta contractions have maxT*maxB rows
        return say("maxT * maxB = %lld rows exceed the contractions' limit of %d", (long long)c->maxT * c->maxB,
                   GEMM_MAX_M);
    if (c->cell != 0 && c->cell != 1) return say("cell %d is neither 0 (clipped ReLU) nor 1 (LSTM)", c->cell);
    if (c->layerNorm != 0 && c->layerNorm != 1)
        return say("layerNorm %d is neither 0 (off) nor 1 (layer normalisation of the ReLU hidden layers)", c->layerNorm);
    if (c->peephole != 0 && c->peephole != 1)
        return say("peephole %d is neither 0 (off) nor 1 (peephole connections of the LSTM cell)", c->peephole);
    if (c->peephole == 1 && c->cell != 1)
        return say("peephole 1 needs the LSTM cell (cell 1); cell is %d", c->cell);
    if (c->layerNorm == 1 && c->layerSize > CTCB_LAYERNORM_MAX_H)
        return say("layerNorm needs layerSize <= %d (the normalisation kernels hold a row on chip); layerSize is %d",
                   CTCB_LAYERNORM_MAX_H, c->layerSize);
    if (c->subsample < 0)
        return say("subsample %d is negative (0 and 1: every layer at the input frame rate; k >= 2: maps subsampleLayer "
                   "and above at 1/k of it)", c->subsample);
    if (c->subsample >= 2) {
        if (c->subsampleLayer < 1 || c->subsampleLayer > c->numLayers + 1)
            return say("subsampleLayer %d is not one of the affine maps 1..%d (numLayers + 1) that subsample %d can "
                       "start at", c->subsampleLayer, c->numLayers + 1, c->subsample);
        const int k = c->subsample, n = c->subsampleLayer == 1 ? c->inputDim : c->layerSize;
        if ((int64_t)k * n > 0x7fffffff || ((int64_t)c->maxT + k - 1) / k * k * c->maxB > 0x7fffffff)
            return say("subsample %d: %d x %d stacked columns or ceil(maxT / k) * k * maxB rows exceed 2^31 - 1", k, k, n);
    }
    if (c->maskFeatDim < 0)
        return say("maskFeatDim %d is negative (0: no input masks; nu > 0: nu filter-bank bins per frame slot)",
                   c->maskFeatDim);
    if (c->maskFeatDim > 0) {
        char why[192];
        if (const char *e = input_mask_layout_error(c->inputDim, c->maskFeatDim, why)) return say("maskFeatDim: %s", e);
    }
    if (c->weightNoise != 0 && c->weightNoise != 1)
        return say("weightNoise %d is neither 0 (off) nor 1 (reserve the noisy copy of the parameters)", c->weightNoise);
    if (c->zoneout != 0 && c->zoneout != 1)
        return say("zoneout %d is neither 0 (off) nor 1 (zoneout of the LSTM cell's state)", c->zoneout);
    if (c->zoneout == 1 && c->cell != 1)
        return say("zoneout 1 needs the LSTM cell (cell 1); cell is %d", c->cell);
    if (c->interLayer != 0) {
        if (c->interLayer < 1 || c->interLayer > c->numLayers - 1)
            return say("interLayer %d is not one of the hidden layers 1..%d (numLayers - 1) an intermediate CTC loss "
                       "can read (0: off)", c->interLayer, c->numLayers - 1);
        if (!(c->interWeight > 0.f && c->interWeight <= 3.4028235e38f))
            return say("interWeight %g of the intermediate CTC loss at layer %d is not a finite value > 0",
                       (double)c->interWeight, c->interLayer);
        if (c->subsample >= 2 && c->subsampleLayer == c->numLayers + 1)
            return say("interLayer %d with subsample %d at subsampleLayer %d (numLayers + 1): the output map then "
                       "reads %d stacked frames and cannot take one layer's output", c->interLayer, c->subsample,
                       c->subsampleLayer, c->subsample);
    }
    if (c->selfCondition != 0 && c->selfCondition != 1)
        return say("selfCondition %d is neither 0 (off) nor 1 (condition the layers above interLayer on its posteriors)",
                   c->selfCondition);
    if (c->selfCondition == 1 && c->interLayer == 0)
        return "selfCondition 1 conditions on the intermediate CTC's posteriors and needs interLayer >= 1; interLayer "
               "is 0";
    if (c->tf32 != 0 && c->tf32 != 1)
        return say("tf32 %d is neither 0 (off) nor 1 (the tensor-core contractions and sweeps in TF32 mode)", c->tf32);
    const bool ok = c->inputDim > 0 && c->outputDim > 1 && c->layerSize > 0 && c->numLayers >= 1 && c->numLayers <= 64 &&
                    c->maxT > 0 && c->maxB > 0 && c->maxLabels >= 0 && c->numTemporal >= 0 &&
                    // a stacked block must lie inside the hidden layers; k <= 1 keeps the silent "no temporal layer" rule below
                    !(c->numTemporal > 1 && (c->temporalLayer <= 0 || c->temporalLayer + c->numTemporal - 1 > c->numLayers));
    if (ok) return nullptr;
    if (c->numTemporal <= 1) return "bad config";
    return say("a block of %d temporal layers from layer %d does not fit in hidden layers 1..%d", c->numTemporal,
               c->temporalLayer, c->numLayers);
}
static int valid_cfg(const ctcb_brnn_config *c) {
    char buf[192];
    return cfg_error(c, buf) == nullptr;
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
// width of layer i of [D, H.., K]
static int layer_size(const ctcb_brnn_config *c, int i) {
    return i == 0 ? c->inputDim : (i <= c->numLayers ? c->layerSize : c->outputDim);
}
// the subsampling factor of a valid config: 1 when off
static int eff_k(const ctcb_brnn_config *c) { return c->subsample >= 2 ? c->subsample : 1; }
// affine map i (1..N+1) and the layer it writes run at the reduced frame rate
static bool is_reduced(const ctcb_brnn_config *c, int i) { return eff_k(c) > 1 && i >= c->subsampleLayer; }
// affine map i reads the stacked frames S of layer i - 1
static bool is_stacked(const ctcb_brnn_config *c, int i) { return eff_k(c) > 1 && i == c->subsampleLayer; }
// columns of affine map i: the width of layer i - 1, k times that where the map reads S
static int map_cols(const ctcb_brnn_config *c, int i) { return (is_stacked(c, i) ? eff_k(c) : 1) * layer_size(c, i - 1); }
static size_t wider_of_H_K(const ctcb_brnn_config *c) {
    return (size_t)(c->layerSize > c->outputDim ? c->layerSize : c->outputDim);
}
static bool is_temporal(const ctcb_brnn_config *c, int i) {
    const int tl = eff_tl(c);
    return tl > 0 && i >= tl && i < tl + eff_nt(c);
}
// G = ndir * 4H: the rows of an LSTM layer's affine map, the pre-activations of the four gates of both directions
static int lstm_rows(const ctcb_brnn_config *c) { return (c->unidirectional ? 1 : 2) * 4 * c->layerSize; }
// rows of affine map i (1..N+1), the width of its output X_i: G at an LSTM layer, else the width of layer i
static int map_rows(const ctcb_brnn_config *c, int i) {
    return (c->cell == 1 && is_temporal(c, i)) ? lstm_rows(c) : layer_size(c, i);
}
// hidden layer i is layer-normalised: a ReLU hidden layer of a layerNorm config (the layers dropout drops)
static bool is_normed(const ctcb_brnn_config *c, int i) {
    return c->layerNorm == 1 && i >= 1 && i <= c->numLayers && !is_temporal(c, i);
}
// the tensors of the flat vector before the [gamma, beta] pairs: the maps, the recurrent matrices and their dummies
static int base_tensors(const ctcb_brnn_config *c) {
    return 2 * (c->numLayers + 1) + eff_nt(c) * (c->unidirectional ? 2 : 4);
}
// flat-vector index of gamma of normalised layer i; beta is the next tensor
static int ln_index(const ctcb_brnn_config *c, int i) {
    int k = 0;
    for (int l = 1; l < i; ++l) k += is_normed(c, l);
    return base_tensors(c) + 2 * k;
}

// the [P, dummy] entries of a peephole net: one per direction of every temporal layer; 0 without
static int peep_tensors(const ctcb_brnn_config *c) {
    return c->peephole == 1 ? eff_nt(c) * (c->unidirectional ? 2 : 4) : 0;
}
// flat-vector index of P of the forward direction of temporal layer j; the backward one, when bi-directional, is two
// tensors behind it.  The entries follow the [gamma, beta] pairs.
static int peep_index(const ctcb_brnn_config *c, int j) {
    return ln_index(c, c->numLayers + 1) + j * (c->unidirectional ? 2 : 4);
}

// the [W_c, b_c] entry of a self-conditioned net, behind everything else; 0 without
static int cond_tensors(const ctcb_brnn_config *c) { return c->selfCondition == 1 ? 2 : 0; }

extern "C" int ctcb_brnn_num_tensors(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    int n = base_tensors(cfg);
    for (int i = 1; i <= cfg->numLayers; ++i) n += 2 * is_normed(cfg, i);
    return n + peep_tensors(cfg) + cond_tensors(cfg);
}

namespace {
// The flat parameter (and gradient) vector of a valid config: W and b of every affine map, then per temporal layer its
// recurrent matrices, each followed by the reference's `dummy` bias (brnnet.py:60-72), then [gamma, beta] of every
// layer-normalised hidden layer, then [P, dummy] of every direction of every peephole LSTM layer, then [W_c, b_c] of a
// self-conditioned net; every tensor 16-byte aligned.
struct NetTable {
    struct Tensor { int64_t off; int32_t rows, cols; };
    int n;
    int nreg;       // tensors 0 .. nreg-1 are the ones L2 regularisation sees (its even ones): all but the LN pairs,
                    // the peephole entries and the conditioning entry
    Tensor t[2 * 65 + 4 * 64 + 2 * 64 + 4 * 64 + 2];
    int64_t params;
    // The gradients that a data-parallel step sums over the ranks early, on the side stream next to the BPTT sweep: the
    // contiguous range from W of the lowest temporal layer to the end of b of layer N+1; empty (at `params`) without a
    // temporal layer.  Everything before and behind it goes with the statistics tail at the end of the step.
    int64_t early_lo, early_hi;
};

void net_table(const ctcb_brnn_config *c, NetTable *nt) {
    const int nl = c->numLayers + 1;
    nt->n = ctcb_brnn_num_tensors(c);
    nt->nreg = base_tensors(c);
    const int cond0 = nt->n - cond_tensors(c), peep0 = cond0 - peep_tensors(c);
    int64_t off = 0;
    for (int t = 0; t < nt->n; ++t) {
        int r, cc;
        if (t >= cond0) {           // W_c (H x K) or b_c (H x 1)
            r = c->layerSize;
            cc = t == cond0 ? c->outputDim : 1;
        } else if (t >= peep0) {           // P (rows i, f, o) of one direction, or its dummy
            r = (t - peep0) % 2 == 0 ? 3 : 1;
            cc = (t - peep0) % 2 == 0 ? c->layerSize : 1;
        } else if (t >= nt->nreg) {        // gamma or beta of a normalised layer
            r = c->layerSize;
            cc = 1;
        } else if (t < 2 * nl) {
            r = map_rows(c, t / 2 + 1);
            cc = (t % 2 == 0) ? map_cols(c, t / 2 + 1) : 1;
        } else if ((t - 2 * nl) % 2 == 0) {
            r = c->cell == 1 ? 4 * c->layerSize : c->layerSize;     // U of an LSTM layer: the four gate blocks
            cc = c->layerSize;
        } else {
            r = cc = 1;
        }
        nt->t[t] = {off, r, cc};
        off += (int64_t)r * cc;
        off = (off + 3) / 4 * 4;   // keep every tensor 16-byte aligned
    }
    nt->params = off;
    nt->early_lo = nt->early_hi = off;
    if (eff_tl(c)) {
        nt->early_lo = nt->t[2 * eff_tl(c)].off;
        nt->early_hi = nt->t[2 * nl - 1].off + c->outputDim;
    }
}
}  // namespace

extern "C" int ctcb_brnn_tensor_info(const ctcb_brnn_config *cfg, int idx, int64_t *offset, int32_t *rows, int32_t *cols) {
    if (!valid_cfg(cfg)) return set_error(CTCB_EINVAL, "ctcb_brnn_tensor_info: bad config");
    NetTable nt;
    net_table(cfg, &nt);
    if (idx < 0 || idx >= nt.n) return set_error(CTCB_EINVAL, "ctcb_brnn_tensor_info: index %d out of range", idx);
    if (offset) *offset = nt.t[idx].off;
    if (rows) *rows = nt.t[idx].rows;
    if (cols) *cols = nt.t[idx].cols;
    return CTCB_OK;
}

extern "C" int64_t ctcb_brnn_param_count(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    NetTable nt;
    net_table(cfg, &nt);
    return nt.params;
}

// ---- the two workspace layouts ------------------------------------------------------------------
namespace {
// The next 256-byte-aligned area behind `off`.  `extent` receives its aligned size: what a callee that is given the
// area with a size gets (the contraction planners choose their splits from it).
size_t take(size_t &off, size_t bytes, size_t *extent = nullptr) {
    const size_t o = off;
    off = align_up(off + bytes, 256);
    if (extent) *extent = off - o;
    return o;
}
// the tail both layouts end with: the sweeps' counters (word 0 the error flag) and their scratch, sized for one plan
struct SweepWs {
    size_t counters, scratch, scratch_bytes;
};
SweepWs take_sweep_ws(size_t &off, const ctcb_brnn_config *c) {
    SweepWs s{};
    s.counters = take(off, sizeof(unsigned int) * 1024);
    // the LSTM sweep's scratch is its dc carry
    s.scratch_bytes = !eff_tl(c) ? 0 : c->cell == 1 ? lstm_carry_bytes(c->layerSize, c->maxB)
                                                    : sweep_tc_workspace_bytes(c->layerSize, c->maxB);
    s.scratch = take(off, s.scratch_bytes);
    return s;
}

struct WsLayout {
    size_t X[66];       // X[1..N] activations, X[N+1] logits
    // For / Back of temporal layer j, and the two dFor / dBack pairs, which consecutive layers alternate (layer j uses
    // pair j % 2); 0 where not laid out
    size_t For[64], Back[64], dFor[2], dBack[2];
    // LSTM layers only: c of each direction, and the output For + Back of a bi-directional layer (X holds its gates)
    size_t Cf[64], Cb[64], Out[64];
    size_t D[67];       // D[j]: gradient w.r.t. the output of affine map j (1..N+1)
    size_t ctc, ctc_bytes;
    size_t gemm, gemm_bytes, gemm2, gemm2_bytes;     // split-K areas of the main chain and of the side stream
    size_t colsum, colsum2, l2_scratch;
    SweepWs sweep;
    // layer-normalised hidden layers only (0 elsewhere): z, and the row statistics of the forward pass; the
    // parameter-gradient partials of the backward pass
    size_t Z[65], Mu[65], Rstd[65], ln_part;
    // subsampling only (0 elsewhere): the stacked input S of map L, its delta dS (L >= 2), T'_u of the call
    size_t S, dS, lens;
    size_t peep_part;   // peephole nets only (0 elsewhere): the partial sums of the peephole weight gradients
    size_t masked;      // maskFeatDim > 0 only (0 elsewhere): the masked copy of the call's features
    size_t noisy;       // weightNoise = 1 only (0 elsewhere): the noisy copy of the parameters
    size_t zo_dh;       // zoneout nets only (0 elsewhere): the BPTT sweep's dh carry
    // interLayer > 0 only (0 elsewhere): the intermediate logits A and D_aux, its nll and skips, and the CTC area it
    // uses (the main one's, unless it runs on more frames)
    size_t inter_A, inter_D, inter_nll, inter_skip, inter_ctc, inter_ctc_bytes;
    size_t cond_X, cond_P, cond_dA;     // selfCondition = 1 only (0 elsewhere): X'_m, P and dA
    size_t total;
};

// rows of the buffers of map / layer i for maxT x maxB: R, or R' = ceil(maxT / k) * maxB from map L up
size_t max_rows(const ctcb_brnn_config *c, int i) {
    return (size_t)(is_reduced(c, i) ? subsampled_frames(c->maxT, eff_k(c)) : c->maxT) * c->maxB;
}
// S: R' x k n floats, n the width of layer L - 1
size_t stacked_bytes(const ctcb_brnn_config *c) {
    return max_rows(c, c->subsampleLayer) * map_cols(c, c->subsampleLayer) * sizeof(float);
}

WsLayout ws_layout(const ctcb_brnn_config *c) {
    WsLayout w{};
    const int N = c->numLayers, H = c->layerSize, nt = eff_nt(c), tl = eff_tl(c);
    const bool uni = (c->unidirectional != 0);
    // H-wide buffers of layer i; the rows only fall from one map to the next, so the lowest user is the largest one
    auto RH = [&](int i) { return max_rows(c, i) * H * sizeof(float); };
    size_t off = 0;
    for (int i = 1; i <= N + 1; ++i) w.X[i] = take(off, max_rows(c, i) * map_rows(c, i) * sizeof(float));
    if (nt) {       // all four for every net with a temporal layer, a uni-directional one too
        w.For[0] = take(off, RH(tl));
        w.Back[0] = take(off, RH(tl));
        w.dFor[0] = take(off, RH(tl));
        w.dBack[0] = take(off, RH(tl));
    }
    // every further temporal layer keeps its own For (and Back): the BPTT masks and the recurrent weight gradients
    // read them.  The dFor / dBack pairs alternate between consecutive layers, so a stack needs one more pair.
    for (int j = 1; j < nt; ++j) {
        w.For[j] = take(off, RH(tl + j));
        if (!uni) w.Back[j] = take(off, RH(tl + j));
    }
    if (nt > 1) {
        w.dFor[1] = take(off, RH(tl + 1));
        if (!uni) w.dBack[1] = take(off, RH(tl + 1));
    }
    const bool lstm = (c->cell == 1);
    for (int j = 0; lstm && j < nt; ++j) {
        w.Cf[j] = take(off, RH(tl + j));
        if (!uni) {
            w.Cb[j] = take(off, RH(tl + j));
            w.Out[j] = take(off, RH(tl + j));
        }
    }
    const size_t wide = wider_of_H_K(c);
    // an LSTM layer's D holds dz, G wide
    const size_t wide_g = lstm && (size_t)lstm_rows(c) > wide ? (size_t)lstm_rows(c) : wide;
    for (int j = 1; j <= N + 1; ++j)
        w.D[j] = take(off, max_rows(c, j) * (map_rows(c, j) == layer_size(c, j) ? wide : wide_g) * sizeof(float));
    w.ctc = take(off, ctcb_ctc_workspace_bytes(c->maxB, (int)(max_rows(c, N + 1) / c->maxB), c->maxLabels), &w.ctc_bytes);
    size_t g = 0;
    auto need = [&](int M_, int N_, int K_) { size_t b = ctcb_gemm_workspace_bytes(M_, N_, K_); if (b > g) g = b; };
    for (int i = 0; i <= N; ++i) {
        const int Ri = (int)max_rows(c, i + 1);     // a valid config: R <= GEMM_MAX_M
        need(Ri, map_rows(c, i + 1), map_cols(c, i + 1));        // forward   X_i . W^T
        need(Ri, map_cols(c, i + 1), map_rows(c, i + 1));        // backward  delta . W
        need(map_rows(c, i + 1), map_cols(c, i + 1), Ri);        // weights   delta^T . X_i
    }
    {                                            // recurrent weight gradients (a pair for the bi-directional layer)
        const size_t b = ctcb_gemm_pair_workspace_bytes(lstm ? 4 * H : H, H, (int)max_rows(c, tl > 0 ? tl : 1));
        if (b > g) g = b;
    }
    w.gemm = take(off, g, &w.gemm_bytes);
    w.gemm2 = take(off, g, &w.gemm2_bytes);
    const size_t R1 = max_rows(c, 1);       // the deltas of map 1, the most rows of any
    w.colsum = take(off, ((R1 + CS_ROWS_MIN - 1) / CS_ROWS_MIN) * wide_g * sizeof(float));
    w.colsum2 = take(off, ((R1 + CS_ROWS_MIN - 1) / CS_ROWS_MIN) * wide_g * sizeof(float));
    w.l2_scratch = take(off, 8192);
    w.sweep = take_sweep_ws(off, c);
    if (c->layerNorm == 1) {
        size_t ln_bytes = layernorm_workspace_bytes((int64_t)max_rows(c, N), H);   // laid out with no normalised layer too
        for (int i = 1; i <= N; ++i) {
            if (!is_normed(c, i)) continue;
            w.Z[i] = take(off, RH(i));
            w.Mu[i] = take(off, max_rows(c, i) * sizeof(float));
            w.Rstd[i] = take(off, max_rows(c, i) * sizeof(float));
            const size_t b = layernorm_workspace_bytes((int64_t)max_rows(c, i), H);
            if (b > ln_bytes) ln_bytes = b;
        }
        w.ln_part = take(off, ln_bytes);
    }
    if (eff_k(c) > 1) {
        w.S = take(off, stacked_bytes(c));
        if (c->subsampleLayer >= 2) w.dS = take(off, stacked_bytes(c));
        w.lens = take(off, (size_t)c->maxB * sizeof(int32_t));
    }
    if (peep_tensors(c))     // the lowest temporal layer has the most rows
        w.peep_part = take(off, lstm_peephole_grad_bytes((int64_t)max_rows(c, tl), H, uni ? 1 : 2));
    if (c->maskFeatDim > 0)     // read by map 1 (its contraction, the frame stacking, its weight gradient) all call long
        w.masked = take(off, (size_t)c->maxT * c->maxB * c->inputDim * sizeof(float));
    if (c->weightNoise == 1)     // read by every stage that reads a weight, all call long
        w.noisy = take(off, (size_t)ctcb_brnn_param_count(c) * sizeof(float));
    if (c->zoneout == 1 && nt)
        w.zo_dh = take(off, lstm_carry_bytes(H, c->maxB));
    if (c->interLayer > 0) {
        const size_t Rm = max_rows(c, c->interLayer), K = (size_t)c->outputDim;
        w.inter_A = take(off, Rm * K * sizeof(float));
        w.inter_D = take(off, Rm * K * sizeof(float));
        w.inter_nll = take(off, (size_t)c->maxB * sizeof(float));
        w.inter_skip = take(off, (size_t)c->maxB * sizeof(int32_t));
        w.inter_ctc = w.ctc;
        w.inter_ctc_bytes = w.ctc_bytes;
        if (Rm > max_rows(c, N + 1))     // below the subsampling point: maxT frames, the main CTC has fewer
            w.inter_ctc = take(off, ctcb_ctc_workspace_bytes(c->maxB, c->maxT, c->maxLabels), &w.inter_ctc_bytes);
    }
    if (c->selfCondition == 1) {
        const size_t Rm = max_rows(c, c->interLayer);
        w.cond_X = take(off, Rm * H * sizeof(float));
        w.cond_P = take(off, Rm * c->outputDim * sizeof(float));
        w.cond_dA = take(off, Rm * c->outputDim * sizeof(float));
    }
    w.total = off;
    return w;
}

// Rows per output tile of both contraction kernels (BM of gemm_simt.cu, TC_BM of gemm_tc.cu): their workspace needs
// change with the row count only at multiples of it.
constexpr int GEMM_ROW_TILE = 128;

// The buffers of a forward-only call: affine map i writes slab i % 2 and reads the other one (or For, the output of
// the uni-directional temporal layer), so two slabs of the largest map output carry the whole stack.  One For (and
// Back, when bi-directional) serves every temporal layer; 0 where not laid out.  Each buffer is sized for the rows of
// the maps that use it (R' from map L up), so a forward-only call fits in the training workspace with subsampling too.
struct FwdLayout {
    size_t slab[2];
    size_t For, Back, gemm, gemm_bytes;
    size_t Cf, Cb, Out;     // LSTM layers: c of each direction and the bi-directional output, shared as For / Back are
    SweepWs sweep;      // as in ws_layout: the same sweep plan
    size_t S, lens;     // subsampling only: the stacked input of map L and T'_u
    size_t cond_A, cond_P;      // selfCondition = 1 only: the intermediate logits A and P
    size_t total;
};

FwdLayout fwd_layout(const ctcb_brnn_config *c) {
    FwdLayout f{};
    const int N = c->numLayers, H = c->layerSize;
    size_t off = 0;
    const bool lstm = (c->cell == 1) && eff_tl(c);
    size_t slab = 0;        // floats: X_i of every map i (its rows x its width; G at an LSTM layer)
    for (int i = 1; i <= N + 1; ++i) {
        const size_t x = max_rows(c, i) * map_rows(c, i);
        if (x > slab) slab = x;
    }
    f.slab[0] = take(off, slab * sizeof(float));
    f.slab[1] = take(off, slab * sizeof(float));
    const size_t R = eff_tl(c) ? max_rows(c, eff_tl(c)) : 0;     // the lowest temporal layer has the most rows
    if (eff_tl(c)) {
        f.For = take(off, R * H * sizeof(float));
        if (!c->unidirectional) f.Back = take(off, R * H * sizeof(float));
    }
    if (lstm) {
        f.Cf = take(off, R * H * sizeof(float));
        if (!c->unidirectional) {
            f.Cb = take(off, R * H * sizeof(float));
            f.Out = take(off, R * H * sizeof(float));
        }
    }
    // ctcb_gemm_f32 takes a smaller plan when its area is short of ctcb_gemm_workspace_bytes(R, ..), and that need is
    // not monotone in R = Tmax*B: below one wave of output tiles the tensor-core plan adds split-K partials.  So that a
    // forward contraction takes, at every R <= maxT*maxB, the plan it takes in the training layout, the area is the
    // largest forward need over all such R, capped at the training area (a contraction that falls back there must
    // fall back here too).  The need changes with R only at multiples of the row tile and grows with R once
    // num_sms() row tiles are exceeded (the split counts are then fixed), so those multiples and R itself bound it.
    // Each map's own rows bound its R (R' from map L up).
    // A self-conditioned net's A and conditioning contractions (R_m x K x H, R_m x H x K) are covered the same way.
    size_t g = 0;
    auto cover = [&](int Rint, int n_out, int n_in) {
        const int Mtop = (Rint < GEMM_ROW_TILE * num_sms()) ? Rint : GEMM_ROW_TILE * num_sms();
        for (int M = GEMM_ROW_TILE; ; M += GEMM_ROW_TILE) {
            const size_t b = ctcb_gemm_workspace_bytes(M <= Mtop ? M : Rint, n_out, n_in);
            if (b > g) g = b;
            if (M > Mtop) break;
        }
    };
    for (int i = 0; i <= N; ++i) cover((int)max_rows(c, i + 1), map_rows(c, i + 1), map_cols(c, i + 1));
    if (c->selfCondition == 1) {
        cover((int)max_rows(c, c->interLayer), c->outputDim, H);
        cover((int)max_rows(c, c->interLayer), H, c->outputDim);
    }
    const size_t train_area = ws_layout(c).gemm_bytes;
    f.gemm = take(off, g < train_area ? g : train_area, &f.gemm_bytes);
    f.sweep = take_sweep_ws(off, c);
    if (eff_k(c) > 1) {     // the slabs ping-pong, and map L - 1 wrote the one map L does not
        f.S = take(off, stacked_bytes(c));
        f.lens = take(off, (size_t)c->maxB * sizeof(int32_t));
    }
    if (c->selfCondition == 1) {
        const size_t RmK = max_rows(c, c->interLayer) * c->outputDim * sizeof(float);
        f.cond_A = take(off, RmK);
        f.cond_P = take(off, RmK);
    }
    f.total = off;
    return f;
}

// Where the forward half reads and writes: X[i] (1..N+1) the output of affine map i (pre-activation, then For+Back,
// at a temporal layer; the logits at N+1), the two sweep outputs of each temporal layer j (one pair shared by all
// layers in the forward-only layout), the split-K area, the sweep counters and scratch.
struct FwdBufs {
    float *X[66];
    float *Z[65], *Mu[65], *Rstd[65];     // normalised layers of a training call: z and the row statistics; else null
    float *For[64], *Back[64];
    float *Cf[64], *Cb[64], *Out[64];     // LSTM layers
    void *gemm;
    size_t gemm_bytes;
    unsigned int *counters;
    void *sweep;
    size_t sweep_bytes;
    float *S;           // subsampling: the stacked input of map L, and T'_u of the call; else null
    int32_t *lens;
    // selfCondition = 1: the intermediate logits A, P, and X'_m (a copy of X_m in a training call; null in a forward-only
    // one, which conditions X_m in place); else null
    float *A, *Pc, *Xc;
};

void fwd_bufs(const FwdLayout &f, int N, int nt, char *ws, FwdBufs *m) {
    for (int i = 1; i <= N + 1; ++i) m->X[i] = (float *)(ws + f.slab[i % 2]);
    for (int j = 0; j < nt; ++j) {     // one pair for every temporal layer: each sweep runs after the last read
        m->For[j] = f.For ? (float *)(ws + f.For) : nullptr;   // offset 0 is slab 0: For / Back were not laid out
        m->Back[j] = f.Back ? (float *)(ws + f.Back) : nullptr;
        m->Cf[j] = f.Cf ? (float *)(ws + f.Cf) : nullptr;
        m->Cb[j] = f.Cb ? (float *)(ws + f.Cb) : nullptr;
        m->Out[j] = f.Out ? (float *)(ws + f.Out) : nullptr;
    }
    m->gemm = ws + f.gemm;
    m->gemm_bytes = f.gemm_bytes;
    m->counters = (unsigned int *)(ws + f.sweep.counters);
    m->sweep = ws + f.sweep.scratch;
    m->sweep_bytes = f.sweep.scratch_bytes;
    m->S = f.S ? (float *)(ws + f.S) : nullptr;
    m->lens = f.S ? (int32_t *)(ws + f.lens) : nullptr;
    m->A = f.cond_A ? (float *)(ws + f.cond_A) : nullptr;
    m->Pc = f.cond_A ? (float *)(ws + f.cond_P) : nullptr;
    m->Xc = nullptr;
}
void train_bufs(const WsLayout &w, int N, int nt, char *ws, FwdBufs *m) {
    for (int i = 1; i <= N + 1; ++i) m->X[i] = (float *)(ws + w.X[i]);
    for (int i = 1; i <= N; ++i) {
        m->Z[i] = w.Z[i] ? (float *)(ws + w.Z[i]) : nullptr;
        m->Mu[i] = w.Z[i] ? (float *)(ws + w.Mu[i]) : nullptr;
        m->Rstd[i] = w.Z[i] ? (float *)(ws + w.Rstd[i]) : nullptr;
    }
    for (int j = 0; j < nt; ++j) {
        m->For[j] = (float *)(ws + w.For[j]);
        m->Back[j] = (float *)(ws + w.Back[j]);      // unused (offset 0) for the uni-directional layers above the first
        m->Cf[j] = (float *)(ws + w.Cf[j]);          // these three: unused (offset 0) unless LSTM
        m->Cb[j] = (float *)(ws + w.Cb[j]);
        m->Out[j] = (float *)(ws + w.Out[j]);
    }
    m->gemm = ws + w.gemm;
    m->gemm_bytes = w.gemm_bytes;
    m->counters = (unsigned int *)(ws + w.sweep.counters);
    m->sweep = ws + w.sweep.scratch;
    m->sweep_bytes = w.sweep.scratch_bytes;
    m->S = w.S ? (float *)(ws + w.S) : nullptr;
    m->lens = w.S ? (int32_t *)(ws + w.lens) : nullptr;
    m->A = w.cond_X ? (float *)(ws + w.inter_A) : nullptr;
    m->Pc = w.cond_X ? (float *)(ws + w.cond_P) : nullptr;
    m->Xc = w.cond_X ? (float *)(ws + w.cond_X) : nullptr;
}
}  // namespace

struct ctcb_brnn {
    ctcb_brnn_config cfg;
    int tl = 0;         // lowest temporal layer or 0
    int nt = 0;         // temporal layers tl .. tl+nt-1 (0 without)
    NetTable net;
    // weight/bias gradients of the layers at and above the temporal layer depend only on their delta, so they
    // run on a side stream next to the (latency-bound, 112-SM) BPTT sweep; created on first use
    cudaStream_t side = nullptr;
    // the main chain of a training call (forward, CTC, delta contractions, sweeps, the tail below the temporal layer)
    // runs on `hi`, forked from the caller's stream and joined back into it: the greatest priority, so its kernels take
    // SMs ahead of the side stream's pending CTAs (the recurrent weight-gradient pair in particular)
    cudaStream_t hi = nullptr;
    // ev_delta[i], temporal layers i only: the deltas of the maps from the last sweep's down to i are complete.
    // ev_sweep: the BPTT sweep of the current temporal layer is queued.
    cudaEvent_t ev_delta[66] = {}, ev_sweep = nullptr;
    cudaEvent_t ev_side = nullptr, ev_fork = nullptr, ev_hi = nullptr;
    // the two dFor/dBack pairs that stacked temporal layers alternate: ev_pair[p] is recorded on the side stream after
    // its last read of pair p, and the BPTT sweep that writes pair p next waits for it
    cudaEvent_t ev_pair[2] = {};
    // selfCondition = 1 with a temporal layer above the conditioned one: dA is complete on main (Step::backward)
    cudaEvent_t ev_cond = nullptr;
    bool side_ready = false;
    // data-parallel callers sum the gradient over ranks first and add reg*W ONCE afterwards (ctcb_brnn_apply_l2_f32);
    // the L2 cost is still reported by every call
    bool defer_l2 = false;
    // data-parallel exchange inside the step (ctcb_brnn_set_comm): the gradients of the layers at and above the temporal
    // layer are summed over ranks on the side stream WHILE the BPTT sweep runs, the rest (+ statistics tail) at the end
    ctcb_comm *comm = nullptr;
    // the forward layout, computed on the first forward-only call (its GEMM area takes a few hundred size queries)
    bool fwd_ready = false;
    FwdLayout fwd;
    // inverted dropout of the ReLU hidden layers in training calls (ctcb_brnn_set_dropout); drop_p == 0: off
    float drop_p = 0.f;
    uint64_t drop_seed = 0;
    const int64_t *drop_step = nullptr;     // the caller's device counter
    uint32_t drop_thr = 0;                  // keep iff Philox output >= drop_thr
    float drop_scale = 1.f;                 // 1 / (1 - p), rounded once; also the delta contraction's alpha
    int64_t drop_first = 0, drop_stride = 1;     // the minibatch index of utterance u, for dropout and the input masks
    // SpecAugment masks of the input features in training calls (ctcb_brnn_set_input_masks); mask_f + mask_t == 0: off
    int mask_f = 0, mask_fw = 0, mask_t = 0, mask_tw = 0;
    double mask_p = 1.0;
    uint64_t mask_seed = 0;
    const int64_t *mask_step = nullptr;
    bool masks_on() const { return mask_f + mask_t > 0; }
    // Gaussian weight noise in training calls (ctcb_brnn_set_weight_noise); noise_sigma == 0: off.  noise_lo / hi: the
    // element ranges of the noised matrices, the even tensors below net.nreg.
    float noise_sigma = 0.f;
    uint64_t noise_seed = 0;
    const int64_t *noise_step = nullptr;
    int noise_n = 0;
    int64_t noise_lo[(2 * 65 + 4 * 64) / 2], noise_hi[(2 * 65 + 4 * 64) / 2];
    bool noise_on() const { return noise_sigma > 0.f; }
    // zoneout of the LSTM layers (ctcb_brnn_set_zoneout); zo_c == zo_h == 0: off, the sweeps without it run
    float zo_c = 0.f, zo_h = 0.f;
    uint64_t zo_seed = 0;
    const int64_t *zo_step = nullptr;
    bool zo_on() const { return zo_c > 0.f || zo_h > 0.f; }
    // the settings of temporal layer i's sweep: the masks in a training call, the expectation in a forward-only one
    LstmZoneout zoneout(int i, bool train, float *dhc) const {
        return LstmZoneout{zo_c, zo_h, train, zo_seed, zo_step, drop_first, drop_stride, i, dhc};
    }

    bool uni() const { return cfg.unidirectional != 0; }
    bool lstm() const { return cfg.cell == 1; }
    int inter() const { return cfg.interLayer; }     // the layer of the intermediate CTC loss, 0 without
    int stats_floats() const { return inter() ? 6 : 4; }     // of stats_out
    int cond() const { return cfg.selfCondition == 1 ? cfg.interLayer : 0; }     // the conditioned layer m, 0 without
    // The early exchange of the data-parallel step (brnn_reduce_early) holds W_{N+1}, b_{N+1}.  A self-conditioned net
    // whose m lies below the lowest temporal layer adds its share of them on main only after the side stream's last
    // weight gradients, so it exchanges the whole gradient at the end instead.
    bool early() const { return tl > 0 && !(cond() && cond() < tl); }
    bool peep() const { return cfg.peephole == 1; }
    int peep_idx(int j) const { return peep_index(&cfg, j); }
    bool temporal(int i) const { return nt > 0 && i >= tl && i < tl + nt; }
    bool normed(int i) const { return is_normed(&cfg, i); }
    bool reduced(int i) const { return is_reduced(&cfg, i); }     // map i runs at 1/k of the input frame rate
    bool stacked(int i) const { return is_stacked(&cfg, i); }     // map i reads S
    int k() const { return eff_k(&cfg); }
    int cols(int i) const { return map_cols(&cfg, i); }           // columns of W_i
    int frames(int i, int Tmax) const { return reduced(i) ? (int)subsampled_frames(Tmax, k()) : Tmax; }
    int size(int i) const { return layer_size(&cfg, i); }
    int rows(int i) const { return map_rows(&cfg, i); }     // width of X_i
    int rec(int j) const { return rec_index(&cfg, j); }
    template <typename T> T *tensor(T *flat, int idx) const { return flat + net.t[idx].off; }
    // activations of layer i as the next layer (and the weight gradients) see them: a uni-directional temporal
    // layer's output IS its forward sweep (rnnet.py:112-116), a bi-directional one's is For + Back (in X_i, or in Out
    // at an LSTM layer, whose X_i holds the gates)
    float *act(const FwdBufs &m, int i) const {
        if (!temporal(i)) return m.X[i];
        return uni() ? m.For[i - tl] : lstm() ? m.Out[i - tl] : m.X[i];
    }
    // what map i + 1 (its contraction, the frame stacking, its weight gradient) reads of layer i: X'_m at the conditioned
    // layer of a training call, else act() (a forward-only call conditions act() in place)
    const float *next_in(const FwdBufs &m, int i) const { return (i == cond() && m.Xc) ? m.Xc : act(m, i); }
    int cond_idx() const { return net.n - 2; }     // flat-vector index of W_c; b_c is the next tensor
};

extern "C" size_t ctcb_brnn_workspace_bytes(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    return ws_layout(cfg).total;
}

extern "C" size_t ctcb_brnn_forward_workspace_bytes(const ctcb_brnn_config *cfg, size_t *error_flag_offset) {
    if (!valid_cfg(cfg)) return 0;
    const FwdLayout f = fwd_layout(cfg);
    if (error_flag_offset) *error_flag_offset = f.sweep.counters;
    return f.total;
}

extern "C" size_t ctcb_brnn_error_flag_offset(const ctcb_brnn_config *cfg) {
    if (!valid_cfg(cfg)) return 0;
    return ws_layout(cfg).sweep.counters;
}

extern "C" int ctcb_brnn_create(const ctcb_brnn_config *cfg, ctcb_brnn **out) {
    char buf[192];
    if (const char *why = cfg_error(cfg, buf)) return set_error(CTCB_EINVAL, "ctcb_brnn_create: %s", why);
    if (!out) return set_error(CTCB_EINVAL, "ctcb_brnn_create: bad config");
    ctcb_brnn *h = new (std::nothrow) ctcb_brnn;
    if (!h) return set_error(CTCB_ENOMEM, "ctcb_brnn_create: out of host memory");
    h->cfg = *cfg;
    if (h->cfg.maxAct <= 0.f) h->cfg.maxAct = 20.0f;   // brnnet.py:32
    h->tl = eff_tl(cfg);
    h->nt = eff_nt(cfg);
    if (h->nt) {      // a width or batch whose sweep the device cannot hold co-resident
        const int ndir = cfg->unidirectional ? 1 : 2;
        Tf32Scope tf32(cfg->tf32);
        // zoneout = 1: the zoneout kernels too, which run whenever a probability is > 0
        int rc = cfg->cell == 1 ? lstm_check(cfg->layerSize, cfg->maxB, ndir, cfg->peephole == 1, false)
                                : sweep_check(cfg->layerSize, cfg->maxB, ndir);
        if (rc == CTCB_OK && cfg->zoneout == 1)
            rc = lstm_check(cfg->layerSize, cfg->maxB, ndir, cfg->peephole == 1, true);
        if (rc != CTCB_OK) {
            char why[512];
            snprintf(why, sizeof(why), "%s", ctcb_last_error());
            delete h;
            return set_error(rc, "ctcb_brnn_create: %s", why);
        }
    }
    net_table(cfg, &h->net);
    for (int idx = 0; idx < h->net.nreg; idx += 2) {     // the matrices ctcb_brnn_apply_l2_f32 regularises
        const NetTable::Tensor &t = h->net.t[idx];
        h->noise_lo[h->noise_n] = t.off;
        h->noise_hi[h->noise_n++] = t.off + (int64_t)t.rows * t.cols;
    }
    *out = h;
    return CTCB_OK;
}

extern "C" void ctcb_brnn_destroy(ctcb_brnn *h) {
    if (h && h->side_ready) {
        cudaStreamDestroy(h->side);
        cudaStreamDestroy(h->hi);
        cudaEventDestroy(h->ev_fork);
        cudaEventDestroy(h->ev_hi);
        for (int i = h->tl; i < h->tl + h->nt; ++i) cudaEventDestroy(h->ev_delta[i]);
        cudaEventDestroy(h->ev_sweep);
        cudaEventDestroy(h->ev_side);
        for (int p = 0; p < 2; ++p) cudaEventDestroy(h->ev_pair[p]);
        if (h->ev_cond) cudaEventDestroy(h->ev_cond);
    }
    delete h;
}

static int ensure_side_stream(ctcb_brnn *h) {
    if (h->side_ready) return CTCB_OK;
    // the lowest priority: the side stream's CTAs never take an SM that a pending sweep cluster could use
    CTCB_CUDA_CHECK(cudaStreamCreateWithPriority(&h->side, cudaStreamNonBlocking, stream_priority_least()));
    for (int i = h->tl; i < h->tl + h->nt; ++i)
        CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_delta[i], cudaEventDisableTiming));
    CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_sweep, cudaEventDisableTiming));
    CTCB_CUDA_CHECK(cudaStreamCreateWithPriority(&h->hi, cudaStreamNonBlocking, stream_priority_greatest()));
    CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_side, cudaEventDisableTiming));
    CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_hi, cudaEventDisableTiming));
    for (int p = 0; p < 2; ++p) CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_pair[p], cudaEventDisableTiming));
    if (h->cond()) CTCB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_cond, cudaEventDisableTiming));
    h->side_ready = true;
    return CTCB_OK;
}

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

extern "C" int ctcb_brnn_sweep_tf32(int mode, int T, int B, int H, const int32_t *T_per_utt, const float *pre,
                                    const float *Wf, const float *Wb, float *outF, float *outB, const float *actF,
                                    const float *actB, float maxAct, void *scratch, size_t scratch_bytes, void *stream) {
    Tf32Scope tf32(1);
    return ctcb_brnn_sweep_f32(mode, T, B, H, T_per_utt, pre, Wf, Wb, outF, outB, actF, actB, maxAct, scratch,
                               scratch_bytes, stream);
}

// ---- the data-parallel exchange: the early range of the net table, then everything else --------------------
static int brnn_reduce_early(ctcb_brnn *h, float *grads, cudaStream_t st) {
    float *pa = grads + h->net.early_lo;
    const int64_t na = h->net.early_hi - h->net.early_lo;
    return comm_allreduce_ranges(h->comm, &pa, &na, 1, st);
}

// The part of the flat gradient that was NOT summed early, plus the statistics tail, in one grouped NCCL launch.
static int brnn_reduce_rest(ctcb_brnn *h, float *grads, float *stats, cudaStream_t st) {
    const int64_t P = h->net.params, lo = h->early() ? h->net.early_lo : P, hi = h->early() ? h->net.early_hi : P;
    float *ptrs[3];
    int64_t cnt[3];
    int k = 0;
    ptrs[k] = grads; cnt[k] = lo; ++k;
    const bool tail_adjacent = (stats == grads + P);
    const int ns = h->stats_floats();
    ptrs[k] = grads + hi; cnt[k] = P - hi + (stats && tail_adjacent ? ns : 0); ++k;
    if (stats && !tail_adjacent) { ptrs[k] = stats; cnt[k] = ns; ++k; }
    return comm_allreduce_ranges(h->comm, ptrs, cnt, k, st);
}

// ---- the step -----------------------------------------------------------------------------------
// brnnet.py:136-173: the affine maps with bias(+ReLU) fused, the two-direction sweep and For+Back at each temporal
// layer, the softmax into probs_out when given.  Clears the sweep error flag first.  drop: a training call with dropout
// on masks the output of every ReLU hidden layer in place right behind its contraction, so the next layer, the weight
// gradients and the ReLU mask of the delta contraction all read the dropped activations.
// With subsampling, map L first stacks its input into S (and T'_u into m.lens); maps L and above run on Tmax' frames.
static int brnn_forward(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt, int B, int Tmax0,
                        const float *params, float *probs_out, const FwdBufs &m, bool train, bool drop,
                        cudaStream_t st) {
    const ctcb_brnn_config &c = h->cfg;
    const int N = c.numLayers, H = c.layerSize, K = c.outputDim;
    const bool uni = h->uni();
    // the sweep kernels' error flag (word 0) is cleared once per call, so a forward-sweep timeout survives the BPTT sweep
    CTCB_CUDA_CHECK(cudaMemsetAsync(m.counters, 0, 16 * sizeof(unsigned int), st));
    for (int i = 1; i <= N + 1; ++i) {
        const float *in = (i == 1) ? feats : h->next_in(m, i - 1);
        const int relu = (i <= N && !h->temporal(i)) ? 1 : 0;
        const int n_out = h->rows(i), n_in = h->cols(i);
        const int Tmax = h->frames(i, Tmax0);
        const int64_t R = (int64_t)Tmax * B;
        const int32_t *Tlen = h->reduced(i) ? m.lens : T_per_utt;
        if (h->stacked(i)) {
            ProfScope ps("subsample", st);
            TRY(run_frame_stack(in, T_per_utt, Tmax0, B, h->size(i - 1), h->k(), m.S, m.lens, st));
            in = m.S;
        }
        // a normalised layer: the contraction writes z (into Z in a training call, in place in the slab otherwise),
        // the normalisation kernel the ReLU output X_i
        const bool ln = h->normed(i);
        float *zi = (ln && m.Z[i]) ? m.Z[i] : m.X[i];
        {
        ProfScope ps("gemm_fwd", st);
        TRY(ctcb_gemm_f32(0, 1, (int)R, n_out, n_in, 1.f, in, n_in, h->tensor(params, 2 * (i - 1)), n_in, 0.f, zi,
                          n_out, h->tensor(params, 2 * (i - 1) + 1), ln ? 0 : relu, nullptr, m.gemm, m.gemm_bytes, st));
        }
        if (ln) {
            const int ig = ln_index(&c, i);
            ProfScope ps("layernorm", st);
            TRY(run_layernorm_forward(zi, m.X[i], m.Mu[i], m.Rstd[i], h->tensor(params, ig), h->tensor(params, ig + 1),
                                      R, n_out, st));
        }
        if (drop && relu) {
            ProfScope ps("dropout", st);
            TRY(run_dropout(m.X[i], R, B, n_out, i, h->drop_seed, h->drop_step, h->drop_first, h->drop_stride,
                            h->drop_thr, h->drop_scale, st));
        }
        if (h->temporal(i) && h->lstm()) {     // the gates over X_i in place, h into For / Back
            const int j = i - h->tl, iU = h->rec(j), iP = h->peep_idx(j);
            const float *Pf = h->peep() ? h->tensor(params, iP) : nullptr;
            const float *Pb = h->peep() && !uni ? h->tensor(params, iP + 2) : nullptr;
            const LstmZoneout zo = h->zoneout(i, train, nullptr);
            {
            ProfScope ps("sweep_fwd", st);
            TRY(run_lstm_sweep(0, Tmax, B, H, Tlen, m.X[i], h->tensor(params, iU),
                               uni ? nullptr : h->tensor(params, iU + 2), Pf, Pb, m.For[j], m.Back[j], m.Cf[j], m.Cb[j],
                               nullptr, nullptr, m.counters, (float *)m.sweep, h->zo_on() ? &zo : nullptr, st));
            }
            if (!uni) {
                ProfScope ps("elementwise", st);
                TRY(run_add2(m.For[j], m.Back[j], m.Out[j], R * H, st));
            }
        } else if (h->temporal(i)) {
            const int j = i - h->tl, iWtf = h->rec(j);
            {
            ProfScope ps("sweep_fwd", st);
            TRY(run_sweep(0, Tmax, B, H, Tlen, m.X[i], h->tensor(params, iWtf),
                          uni ? nullptr : h->tensor(params, iWtf + 2), m.For[j], m.Back[j], nullptr, nullptr, c.maxAct,
                          m.counters, m.sweep, m.sweep_bytes, st));
            }
            if (!uni) {     // over the pre-activation, which nothing reads after the sweep
                ProfScope ps("elementwise", st);
                TRY(run_add2(m.For[j], m.Back[j], m.X[i], R * H, st));     // brnnet.py:153
            }
        }
        if (i == h->cond()) {     // A, P = softmax(A), X'_m = X_m + P W_c^T + b_c (include/ctcb200.h: selfCondition)
            const float *Wc = h->tensor(params, h->cond_idx()), *bc = h->tensor(params, h->cond_idx() + 1);
            float *Xm = h->act(m, i);
            ProfScope ps("self_cond", st);
            TRY(ctcb_gemm_f32(0, 1, (int)R, K, H, 1.f, Xm, H, h->tensor(params, 2 * N), H, 0.f, m.A, K,
                              h->tensor(params, 2 * N + 1), 0, nullptr, m.gemm, m.gemm_bytes, st));
            TRY(run_softmax_rows(m.A, m.Pc, R, K, st));
            if (m.Xc) {     // a training call keeps X_m (the masks, the head, the BPTT) and conditions a copy
                CTCB_CUDA_CHECK(cudaMemcpyAsync(m.Xc, Xm, (size_t)R * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
                Xm = m.Xc;
            }
            TRY(ctcb_gemm_f32(0, 1, (int)R, H, K, 1.f, m.Pc, K, Wc, K, 1.f, Xm, H, bc, 0, nullptr, m.gemm, m.gemm_bytes,
                              st));
        }
    }
    if (probs_out) TRY(run_softmax_rows(m.X[N + 1], probs_out, (int64_t)h->frames(N + 1, Tmax0) * B, K, st));
    return CTCB_OK;
}

namespace {
// What the stages of one training call share: the handle, the forward half's buffers `m`, the layout `w` of the
// workspace `ws` for what only the backward half uses, the call's arguments.  `main` carries the forward pass, the
// CTC, the delta chain and the sweeps, `side` the weight gradients of the layers at and above the lowest temporal
// layer; `caller` is the stream the call was given, which `main` is forked from and both are joined into.  Without a
// temporal layer main == caller and there is no side stream.  `params` is what every stage reads (the noisy copy with
// weight noise on), `clean` the caller's vector, which only the L2 term reads.
struct Step {
    ctcb_brnn *h;
    const FwdBufs &m;
    const WsLayout &w;
    char *ws;
    const float *feats, *params, *clean;
    const int32_t *T_per_utt;
    float *grads;
    int B, Tmax;            // Tmax of the input; map i runs on T(i) frames
    bool first, last;       // CTCB_PART_FIRST: overwrite the gradients, else add to them; CTCB_PART_LAST: exchange and L2
    bool drop, dp;
    cudaStream_t main, side, caller;

    float *buf(size_t off) const { return (float *)(ws + off); }
    const float *P(int idx) const { return h->tensor(params, idx); }
    float *G(int idx) const { return h->tensor(grads, idx); }
    float beta_g() const { return first ? 0.f : 1.f; }      // weight-gradient contractions: C = dW (+ C)
    // frames, rows and frame counts of map / layer i: Tmax' and T'_u from map L up when subsampled
    int T(int i) const { return h->frames(i, Tmax); }
    int64_t R(int i) const { return (int64_t)T(i) * B; }
    const int32_t *lens(int i) const { return h->reduced(i) ? m.lens : T_per_utt; }
    // the delta of map i; rnnet.py:162-177: the BPTT result of a uni-directional layer is the delta
    // (an LSTM layer's BPTT writes its dz, the delta of its map, into D)
    float *delta(int i) const {
        return buf((h->uni() && h->temporal(i + 1) && !h->lstm()) ? w.dFor[(i + 1 - h->tl) % 2] : w.D[i + 1]);
    }
    int weight_grads(int i, bool on_side) const;
    int head_grads(bool on_side) const;
    int cond_backward(int i, float *doth, float alpha) const;
    int rec_weight_grads(int j) const;
    int backward() const;
    int finish(float *stats, float *regcost_out) const;
};
}  // namespace

// the weight and bias gradients of map i, on the side stream or in the main chain, where its delta is complete
int Step::weight_grads(int i, bool on_side) const {
    const cudaStream_t st = on_side ? side : main;
    const float *Xi = h->stacked(i + 1) ? m.S : (i == 0) ? feats : h->next_in(m, i);
    const int n_out = h->rows(i + 1), n_in = h->cols(i + 1);
    // dW = delta^T . X_i   (brnnet.py:196); dW_L = delta^T . S
    {
    ProfScope ps("gemm_dw", st);
    TRY(ctcb_gemm_f32(1, 0, n_out, n_in, (int)R(i + 1), 1.f, delta(i), n_out, Xi, n_in, beta_g(), G(2 * i), n_in, nullptr,
                      0, nullptr, on_side ? ws + w.gemm2 : m.gemm, on_side ? w.gemm2_bytes : m.gemm_bytes, st));
    }
    // db = row sums of delta   (brnnet.py:200)
    {
    ProfScope ps("colsum", st);
    TRY(run_colsum(delta(i), R(i + 1), n_out, buf(on_side ? w.colsum2 : w.colsum), G(2 * i + 1), !first, st));
    }
    // the intermediate loss's share of W_{N+1} and b_{N+1}: added behind the main one on the same stream, so ahead of
    // the early exchange, whose range holds them.  The side stream gets here behind ev_delta, which main records after
    // the intermediate CTC (and, self-conditioned with m at or above the highest temporal layer, after layer m's stage,
    // which completes dA).  A self-conditioned net with m below the highest temporal layer adds it at layer m
    // (Step::cond_backward).
    if (i == h->cfg.numLayers && h->inter() && (!h->cond() || (h->tl > 0 && h->cond() >= h->tl + h->nt - 1)))
        TRY(head_grads(on_side));
    if (h->uni() && h->temporal(i + 1) && !h->lstm() && i + 1 - h->tl >= 2)  // the last read of the pair of uni-directional layer i + 1
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_pair[(i + 1 - h->tl) % 2], side));
    // every gradient tensor of the layers >= tl is now queued on the side stream: sum that contiguous range over
    // the ranks there, next to the BPTT sweep on the main stream
    if (dp && last && on_side && i == h->tl && h->early()) TRY(brnn_reduce_early(h, grads, side));
    return CTCB_OK;
}

// dW_{N+1} += D^T X_m, db_{N+1} += the column sums of D, behind the main term: D = D_aux, or dA when self-conditioned
int Step::head_grads(bool on_side) const {
    const cudaStream_t st = on_side ? side : main;
    const int N = h->cfg.numLayers, mi = h->inter(), K = h->cfg.outputDim, H = h->cfg.layerSize;
    const float *D = buf(h->cond() ? w.cond_dA : w.inter_D);
    ProfScope ps("inter_ctc_dw", st);
    TRY(ctcb_gemm_f32(1, 0, K, H, (int)R(mi), 1.f, D, K, h->act(m, mi), H, 1.f, G(2 * N), H, nullptr, 0, nullptr,
                      on_side ? ws + w.gemm2 : m.gemm, on_side ? w.gemm2_bytes : m.gemm_bytes, st));
    TRY(run_colsum(D, R(mi), K, buf(on_side ? w.colsum2 : w.colsum), G(2 * N + 1), true, st));
    return CTCB_OK;
}

// Self-conditioned layer i = m (include/ctcb200.h: selfCondition), on main: doth holds D'_m, the unmasked delta of map
// m + 1 at layer m's rate.  dP = D'_m W_c into the dA buffer, dW_c and db_c (before doth is overwritten), dA in place,
// then doth = alpha [X_m > 0] (D'_m + dA W_{N+1}).  Where dA's share of W_{N+1}, b_{N+1} goes, so that it lands behind
// weight_grads(N)'s writes and ahead of the early exchange: inside weight_grads(N) when m is at or above the highest
// temporal layer; on main here without a temporal layer; otherwise on the side stream here, behind ev_cond (host order
// puts it after weight_grads(N), enqueued in an earlier iteration, and ahead of this iteration's weight gradients and
// the early exchange, which early() drops when m is below the lowest temporal layer).
int Step::cond_backward(int i, float *doth, float alpha) const {
    const int N = h->cfg.numLayers, K = h->cfg.outputDim, H = h->cfg.layerSize, ic = h->cond_idx();
    const int64_t Rm = R(i);
    float *dA = buf(w.cond_dA);
    {
    ProfScope ps("self_cond_bwd", main);
    TRY(ctcb_gemm_f32(0, 0, (int)Rm, K, H, 1.f, doth, H, P(ic), K, 0.f, dA, K, nullptr, 0, nullptr, m.gemm,
                      m.gemm_bytes, main));
    TRY(ctcb_gemm_f32(1, 0, H, K, (int)Rm, 1.f, doth, H, m.Pc, K, beta_g(), G(ic), K, nullptr, 0, nullptr, m.gemm,
                      m.gemm_bytes, main));
    TRY(run_colsum(doth, Rm, H, buf(w.colsum), G(ic + 1), !first, main));
    TRY(run_softmax_rows_backward(m.Pc, dA, buf(w.inter_D), dA, Rm, K, main));
    TRY(ctcb_gemm_f32(0, 0, (int)Rm, H, K, alpha, dA, K, P(2 * N), H, alpha, doth, H, nullptr, 0,
                      h->temporal(i) ? nullptr : h->act(m, i), m.gemm, m.gemm_bytes, main));
    }
    if (h->tl == 0) return head_grads(false);
    if (i >= h->tl + h->nt - 1) return CTCB_OK;
    CTCB_CUDA_CHECK(cudaEventRecord(h->ev_cond, main));
    TRY(stall(main, STALL_MAIN));
    CTCB_CUDA_CHECK(cudaStreamWaitEvent(side, h->ev_cond, 0));
    TRY(stall(side, STALL_SIDE));
    return head_grads(true);
}

// The recurrent weight gradients of temporal layer j (brnnet.py:227-230), behind its BPTT sweep: independent of the
// rest of the backward pass, so they go to the side stream as well.
int Step::rec_weight_grads(int j) const {
    const int H = h->cfg.layerSize, iWtf = h->rec(j), iWtb = iWtf + 2;
    float *dFor = buf(w.dFor[j % 2]), *dBack = buf(w.dBack[j % 2]);
    CTCB_CUDA_CHECK(cudaEventRecord(h->ev_sweep, main));
    TRY(stall(main, STALL_MAIN));
    CTCB_CUDA_CHECK(cudaStreamWaitEvent(side, h->ev_sweep, 0));
    TRY(stall(side, STALL_SIDE));
    ProfScope ps("gemm_dw_rec", side);
    const int Tmax = T(h->tl + j);
    const int64_t R = this->R(h->tl + j);
    if (h->lstm()) {     // dU = sum_t dz_t h_prev^T: the dz of both directions lie side by side in the layer's D, G wide
        const int ldz = h->rows(h->tl + j), M = 4 * H;
        const float *dz = buf(w.D[h->tl + j]);
        if (Tmax > 1) {
            const int64_t Rm = R - B;
            if (h->uni())
                TRY(ctcb_gemm_f32(1, 0, M, H, (int)Rm, 1.f, dz + (int64_t)B * ldz, ldz, m.For[j], H, beta_g(), G(iWtf), H,
                                  nullptr, 0, nullptr, ws + w.gemm2, w.gemm2_bytes, side));
            else
                TRY(ctcb_gemm_pair_f32(1, 0, M, H, (int)Rm, 1.f, dz + (int64_t)B * ldz, dz + M, ldz, m.For[j],
                                       m.Back[j] + (int64_t)B * H, H, beta_g(), G(iWtf), G(iWtb), H, ws + w.gemm2,
                                       w.gemm2_bytes, side));
        } else if (first) {
            CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtf), 0, sizeof(float) * M * H, side));
            if (!h->uni()) CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtb), 0, sizeof(float) * M * H, side));
        }
        if (h->peep()) {     // dP = sums of dz . c over the rows (one frame has dp_o too), in this phase's profile
            const int iP = h->peep_idx(j);
            TRY(run_lstm_peephole_grad(Tmax, B, H, dz, m.Cf[j], h->uni() ? nullptr : m.Cb[j], G(iP),
                                       h->uni() ? nullptr : G(iP + 2), !first, buf(w.peep_part), side));
        }
    } else if (Tmax > 1) {
        const int64_t Rm = R - B;
        if (h->uni())
            TRY(ctcb_gemm_f32(1, 0, H, H, (int)Rm, 1.f, dFor + (int64_t)B * H, H, m.For[j], H, beta_g(), G(iWtf), H,
                              nullptr, 0, nullptr, ws + w.gemm2, w.gemm2_bytes, side));
        else     // both directions in one launch
            TRY(ctcb_gemm_pair_f32(1, 0, H, H, (int)Rm, 1.f, dFor + (int64_t)B * H, dBack, H, m.For[j],
                                   m.Back[j] + (int64_t)B * H, H, beta_g(), G(iWtf), G(iWtb), H, ws + w.gemm2,
                                   w.gemm2_bytes, side));
    } else if (first) {     // one frame: no recurrence, nothing to add to earlier micro-batches
        CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtf), 0, sizeof(float) * H * H, side));
        if (!h->uni()) CTCB_CUDA_CHECK(cudaMemsetAsync(G(iWtb), 0, sizeof(float) * H * H, side));
    }
    return CTCB_OK;
}

// brnnet.py:188-243.  Per temporal layer from the top: the delta GEMM without a mask, the BPTT sweep into pair j % 2,
// then on the side stream the weight gradients of the maps from the last sweep's down to this layer and the recurrent
// weight-gradient pair, add2.  The side stream's weight gradients become ready together with the sweep, not before
// it: the sweep's clusters (the higher priority) take their SMs first and the GEMMs run on the rest for the length
// of the sweep, instead of holding SMs the sweep then waits for.  Layer j - 2 writes the pair layer j used: its
// sweep waits for ev_pair, recorded on the side stream behind the last read of that pair (the recurrent weight
// gradients; for a uni-directional layer the weight gradient of the map above, whose delta the pair is).
int Step::backward() const {
    const int N = h->cfg.numLayers, H = h->cfg.layerSize, tl = h->tl, nt = h->nt;
    const bool uni = h->uni();
    int side_top = N;      // the highest map >= tl whose weight gradients are not queued yet
    for (int i = N; i >= 0; --i) {
        // layers i >= tl > 0: dW/db on the side stream, delta chain + BPTT on the main one
        if (!(tl > 0 && i >= tl)) TRY(weight_grads(i, false));
        if (i == 0) break;
        const int n_out = h->rows(i + 1), n_in = h->cols(i + 1), n = h->size(i);
        const int64_t R = this->R(i);
        // an LSTM layer's dh goes to the pair; its BPTT writes dz into D[i]
        const bool lstm = h->temporal(i) && h->lstm();
        float *doth = buf(lstm ? w.dFor[(i - tl) % 2] : w.D[i]);
        // below map L the contraction writes dS, in the layout of S, and dS is unstacked into doth
        const bool stacked = h->stacked(i + 1);
        // delta <- delta . W, with the ReLU mask sign(hActs[i]) fused (brnnet.py:203-204,235-237).  A dropped
        // layer's X_i is 0 at every dropped unit, so the same mask removes those; the kept ones were scaled by
        // drop_scale in the forward pass, and so is their delta, through alpha.  S holds X_i stacked, and 0 at the
        // padding frames, whose delta is 0 either way.
        // The self-conditioned layer takes D'_m without the mask and alpha, which cond_backward applies.
        const bool cond = (i == h->cond());
        const float *mask = (h->temporal(i) || cond) ? nullptr : stacked ? m.S : h->act(m, i);
        const float alpha = (drop && !h->temporal(i)) ? h->drop_scale : 1.f;
        {
        ProfScope ps("gemm_delta", main);
        TRY(ctcb_gemm_f32(0, 0, (int)this->R(i + 1), n_in, n_out, cond ? 1.f : alpha, delta(i), n_out, P(2 * i), n_in,
                          0.f, stacked ? buf(w.dS) : doth, n_in, nullptr, 0, mask, m.gemm, m.gemm_bytes, main));
        }
        if (stacked) {
            ProfScope ps("subsample", main);
            TRY(run_frame_unstack(buf(w.dS), T_per_utt, T(i), B, n, h->k(), doth, main));
        }
        if (cond) {
            TRY(cond_backward(i, doth, alpha));
        } else if (i == h->inter()) {     // + D_aux W_{N+1}, at layer i's own rate, under the same mask and alpha
            ProfScope ps("inter_ctc_delta", main);
            TRY(ctcb_gemm_f32(0, 0, (int)R, n, h->cfg.outputDim, alpha, buf(w.inter_D), h->cfg.outputDim, P(2 * N), n,
                              1.f, doth, n, nullptr, 0, h->temporal(i) ? nullptr : h->act(m, i), m.gemm, m.gemm_bytes,
                              main));
        }
        if (h->normed(i)) {     // g -> dz in place, before anything reads D[i]; dgamma / dbeta of the layer
            const int ig = ln_index(&h->cfg, i);
            ProfScope ps("layernorm", main);
            TRY(run_layernorm_backward(doth, m.Z[i], m.Mu[i], m.Rstd[i], P(ig), G(ig), G(ig + 1), R, n, !first,
                                       buf(w.ln_part), main));
        }
        if (!h->temporal(i)) continue;
        // brnnet.py:207-233
        const int j = i - tl, p = j % 2, iWtf = h->rec(j);
        if (j + 2 < nt && !lstm)      // layer j + 2 used this pair (an LSTM layer's pair is read on this stream only)
            CTCB_CUDA_CHECK(cudaStreamWaitEvent(main, h->ev_pair[p], 0));
        // the deltas of maps side_top..i are complete here
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_delta[i], main));
        TRY(stall(main, STALL_MAIN));
        {
        ProfScope ps("sweep_bptt", main);
        if (lstm) {
            const LstmZoneout zo = h->zoneout(i, true, buf(w.zo_dh));
            TRY(run_lstm_sweep(1, T(i), B, H, lens(i), m.X[i], P(iWtf), uni ? nullptr : P(iWtf + 2),
                               h->peep() ? P(h->peep_idx(j)) : nullptr,
                               h->peep() && !uni ? P(h->peep_idx(j) + 2) : nullptr, nullptr, nullptr, m.Cf[j], m.Cb[j],
                               doth, buf(w.D[i]), m.counters, (float *)m.sweep, h->zo_on() ? &zo : nullptr, main));
        } else
            TRY(run_sweep(1, T(i), B, H, lens(i), doth, P(iWtf), uni ? nullptr : P(iWtf + 2), buf(w.dFor[p]),
                          buf(w.dBack[p]), m.For[j], m.Back[j], h->cfg.maxAct, m.counters, m.sweep, m.sweep_bytes, main));
        }
        CTCB_CUDA_CHECK(cudaStreamWaitEvent(side, h->ev_delta[i], 0));
        TRY(stall(side, STALL_SIDE));
        for (; side_top >= i; --side_top) TRY(weight_grads(side_top, true));
        TRY(rec_weight_grads(j));
        if (!uni && !lstm) {
            if (j >= 2) CTCB_CUDA_CHECK(cudaEventRecord(h->ev_pair[p], side));
            TRY(run_add2(buf(w.dFor[p]), buf(w.dBack[p]), doth, R * H, main));
        }
    }
    // the main stream's tail writes nothing the side stream touches, so it runs next to the recurrent weight gradients
    for (int j = 0; j < nt; ++j) {   // the `dummy` biases never receive gradient
        CTCB_CUDA_CHECK(cudaMemsetAsync(G(h->rec(j) + 1), 0, sizeof(float), main));
        if (!uni) CTCB_CUDA_CHECK(cudaMemsetAsync(G(h->rec(j) + 3), 0, sizeof(float), main));
        if (h->peep()) {
            CTCB_CUDA_CHECK(cudaMemsetAsync(G(h->peep_idx(j) + 1), 0, sizeof(float), main));
            if (!uni) CTCB_CUDA_CHECK(cudaMemsetAsync(G(h->peep_idx(j) + 3), 0, sizeof(float), main));
        }
    }
    return CTCB_OK;
}

// What only the last micro-batch of a step does, on the caller's stream behind the join: the rest of the exchange and
// the L2 term (brnnet.py:177-183,197-198,244-247).
int Step::finish(float *stats, float *regcost_out) const {
    const float reg = h->cfg.reg;
    if (dp) TRY(brnn_reduce_rest(h, grads, stats, caller));
    if (regcost_out) {
        set_scalar_kernel<<<1, 1, 0, caller>>>(regcost_out, 0.f);
        CTCB_LAUNCH_CHECK();
    }
    if (!h->defer_l2) TRY(ctcb_brnn_apply_l2_f32(h, clean, grads, caller));
    if (regcost_out && reg > 0.f)
        for (int idx = 0; idx < h->net.nreg; idx += 2) {     // the same weight matrices
            const NetTable::Tensor &t = h->net.t[idx];
            TRY(run_sumsq(clean + t.off, (int64_t)t.rows * t.cols, regcost_out, 0.5f * reg, 1, ws + w.l2_scratch, caller));
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
    const ctcb_brnn_config &c = h->cfg;
    Tf32Scope tf32(c.tf32);     // every contraction and sweep this call plans, training or forward-only
    if (B <= 0 || B > c.maxB || Tmax <= 0 || Tmax > c.maxT)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: batch %d x %d frames exceeds the configured %d x %d",
                         B, Tmax, c.maxB, c.maxT);
    const bool train = (grads != nullptr);
    if (train && (!labels || !label_off || !cost_out || !skip_out))
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: training mode needs labels and cost/skip outputs");
    if (!train && !probs_out)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: forward-only mode needs probs_out");
    if (train && h->zo_on() && !h->zo_step)
        return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: zoneout (zc = %g, zh = %g) in a training call needs a "
                         "step counter (ctcb_brnn_set_zoneout)", (double)h->zo_c, (double)h->zo_h);
    const cudaStream_t caller = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    const int N = c.numLayers, K = c.outputDim;
    const int64_t R = (int64_t)Tmax * B;
    if (R > 0x7fffffff) return set_error(CTCB_EINVAL, "ctcb_brnn_cost_and_grad: T*B too large");
    if (!train) {     // the forward layout whatever the size given: the same kernels and plans as a training call
        if (!h->fwd_ready) {
            h->fwd = fwd_layout(&c);
            h->fwd_ready = true;
        }
        if (!workspace || ws_bytes < h->fwd.total)
            return set_error(CTCB_ENOMEM, "ctcb_brnn_cost_and_grad: workspace %zu < %zu bytes", ws_bytes, h->fwd.total);
        FwdBufs m{};
        fwd_bufs(h->fwd, N, h->nt, ws, &m);
        return brnn_forward(h, feats, T_per_utt, B, Tmax, params, probs_out, m, false, false, caller);
    }
    // planned on every call: the contraction planners' overrides may change under a live handle (common.cuh)
    const WsLayout w = ws_layout(&c);
    if (!workspace || ws_bytes < w.total)
        return set_error(CTCB_ENOMEM, "ctcb_brnn_cost_and_grad: workspace %zu < %zu bytes", ws_bytes, w.total);
    FwdBufs m{};
    train_bufs(w, N, h->nt, ws, &m);
    const bool dp = (h->comm != nullptr) && comm_world(h->comm) > 1;
    // with input masks on, every stage of the call reads the masked copy in place of feats, which it never writes
    const float *in = h->masks_on() ? (const float *)(ws + w.masked) : feats;
    // with weight noise on, every stage reads the noisy copy in place of params; the L2 term reads params
    const float *wts = h->noise_on() ? (const float *)(ws + w.noisy) : params;
    Step s{h, m, w, ws, in, wts, params, T_per_utt, grads, B, Tmax, first, last, h->drop_p > 0.f, dp,
           caller, nullptr, caller};
    const bool overlap = (h->tl > 0);
    if (overlap) {     // fork: the main chain runs on h->hi until the join below
        TRY(ensure_side_stream(h));
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_fork, caller));
        CTCB_CUDA_CHECK(cudaStreamWaitEvent(h->hi, h->ev_fork, 0));
        TRY(stall(h->hi, STALL_MAIN));
        s.main = h->hi;
        s.side = h->side;
    }
    if (h->masks_on()) {     // the side stream reads the copy only behind events recorded on main after this
        ProfScope ps("input_mask", s.main);
        TRY(run_input_mask(feats, T_per_utt, B, Tmax, c.inputDim, c.maskFeatDim, h->mask_f, h->mask_fw, h->mask_t,
                           h->mask_tw, h->mask_p, h->mask_seed, h->mask_step, h->drop_first, h->drop_stride,
                           (float *)(ws + w.masked), s.main));
    }
    if (h->noise_on()) {     // the side stream reads no weight; it meets main only behind events recorded after this
        ProfScope ps("weight_noise", s.main);
        TRY(run_weight_noise(params, (float *)(ws + w.noisy), h->net.params, h->noise_lo, h->noise_hi, h->noise_n,
                             h->noise_sigma, h->noise_seed, h->noise_step, s.main));
    }
    TRY(brnn_forward(h, in, T_per_utt, B, Tmax, wts, probs_out, m, true, s.drop, s.main));
    {     // brnnet.py:161-175
    ProfScope ps("ctc", s.main);
    TRY(ctcb_ctc_loss_grad_f32(m.X[N + 1], 0, (int64_t)K, (int64_t)B * K, labels, label_off, s.lens(N + 1), B, s.T(N + 1), K,
                               c.maxLabels, 0, s.buf(w.D[N + 1]), cost_out, skip_out, ws + w.ctc, w.ctc_bytes, s.main));
    }
    float *inter_nll = h->inter() ? s.buf(w.inter_nll) : nullptr;
    int32_t *inter_skip = h->inter() ? (int32_t *)(ws + w.inter_skip) : nullptr;
    if (h->inter()) {     // A = X_m W_{N+1}^T + b_{N+1}, its CTC, and D_aux = lambda dnll/dA scaled in place: the two
                          // contractions and the column sums of the backward pass then read the same values
        const int mi = h->inter(), H = c.layerSize;
        float *A = s.buf(w.inter_A), *Da = s.buf(w.inter_D);
        ProfScope ps("inter_ctc", s.main);
        if (!h->cond())     // a self-conditioned net computed A in the forward pass
            TRY(ctcb_gemm_f32(0, 1, (int)s.R(mi), K, H, 1.f, h->act(m, mi), H, s.P(2 * N), H, 0.f, A, K, s.P(2 * N + 1),
                              0, nullptr, m.gemm, m.gemm_bytes, s.main));
        TRY(ctcb_ctc_loss_grad_f32(A, 0, (int64_t)K, (int64_t)B * K, labels, label_off, s.lens(mi), B, s.T(mi), K,
                                   c.maxLabels, 0, Da, inter_nll, inter_skip, ws + w.inter_ctc, w.inter_ctc_bytes,
                                   s.main));
        TRY(run_scale(Da, s.R(mi) * K, c.interWeight, s.main));
    }
    TRY(s.backward());
    if (stats_out)     // after both sweeps, so that the tail carries the error flag of either
        TRY(run_batch_stats(cost_out, skip_out, B, stats_out, m.counters, !first, s.main));
    if (stats_out && h->inter()) TRY(run_inter_stats(inter_nll, inter_skip, B, stats_out + 4, !first, s.main));
    if (overlap) {     // join: every gradient tensor is complete on the caller's stream from here on
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_side, h->side));
        CTCB_CUDA_CHECK(cudaEventRecord(h->ev_hi, h->hi));
        CTCB_CUDA_CHECK(cudaStreamWaitEvent(caller, h->ev_side, 0));
        CTCB_CUDA_CHECK(cudaStreamWaitEvent(caller, h->ev_hi, 0));
    }
    // an earlier micro-batch of the step: the exchange and the L2 term wait for the sum of all of them
    return last ? s.finish(stats_out, regcost_out) : CTCB_OK;
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
    if (h->cfg.reg <= 0.f) return CTCB_OK;
    for (int idx = 0; idx < h->net.nreg; idx += 2) {     // weight matrices only, as brnnet.py:197-198,244-247
        const NetTable::Tensor &t = h->net.t[idx];
        TRY(ctcb_axpy_f32(grads + t.off, params + t.off, h->cfg.reg, (int64_t)t.rows * t.cols, stream));
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
    if (h->early()) TRY(brnn_reduce_early(h, grads, (cudaStream_t)stream));
    TRY(brnn_reduce_rest(h, grads, stats_out, (cudaStream_t)stream));
    return h->defer_l2 ? CTCB_OK : ctcb_brnn_apply_l2_f32(h, params, grads, stream);
}

extern "C" int ctcb_brnn_set_dropout(ctcb_brnn *h, float p, uint64_t seed, const int64_t *step) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_dropout: null handle");
    if (!(p >= 0.f && p < 1.f)) return set_error(CTCB_EINVAL, "ctcb_brnn_set_dropout: p = %g is not in [0, 1)", (double)p);
    if (p > 0.f && !step) return set_error(CTCB_EINVAL, "ctcb_brnn_set_dropout: p = %g needs a step counter", (double)p);
    const double pd = (double)p;
    h->drop_p = p;
    h->drop_seed = seed;
    h->drop_step = step;
    h->drop_thr = (uint32_t)std::floor(pd * 4294967296.0);     // < 2^32: p <= 1 - 2^-24
    h->drop_scale = (float)(1.0 / (1.0 - pd));
    return CTCB_OK;
}

extern "C" int ctcb_brnn_set_dropout_utts(ctcb_brnn *h, int64_t first, int64_t stride) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_dropout_utts: null handle");
    if (first < 0 || stride < 1)
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_dropout_utts: first = %lld, stride = %lld (need first >= 0, "
                         "stride >= 1)", (long long)first, (long long)stride);
    h->drop_first = first;
    h->drop_stride = stride;
    return CTCB_OK;
}

extern "C" int ctcb_brnn_set_input_masks(ctcb_brnn *h, int freqMasks, int freqWidth, int timeMasks, int timeWidth,
                                         double timeRatio, uint64_t seed, const int64_t *step) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_input_masks: null handle");
    char buf[192];
    if (const char *why = input_mask_policy_error(h->cfg.maskFeatDim, freqMasks, freqWidth, timeMasks, timeWidth,
                                                  timeRatio, buf))
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_input_masks: %s", why);
    if (freqMasks + timeMasks > 0 && !step)
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_input_masks: %d frequency and %d time masks need a step counter",
                         freqMasks, timeMasks);
    h->mask_f = freqMasks;
    h->mask_fw = freqWidth;
    h->mask_t = timeMasks;
    h->mask_tw = timeWidth;
    h->mask_p = timeRatio;
    h->mask_seed = seed;
    h->mask_step = step;
    return CTCB_OK;
}

extern "C" int ctcb_brnn_set_weight_noise(ctcb_brnn *h, float sigma, uint64_t seed, const int64_t *step) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_weight_noise: null handle");
    if (!(sigma >= 0.f && sigma <= 3.4028235e38f))
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_weight_noise: sigma = %g is not a finite value >= 0", (double)sigma);
    if (sigma > 0.f && h->cfg.weightNoise != 1)
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_weight_noise: sigma = %g needs the noisy copy (weightNoise = 1 in "
                         "the config)", (double)sigma);
    if (sigma > 0.f && !step)
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_weight_noise: sigma = %g needs a step counter", (double)sigma);
    h->noise_sigma = sigma;
    h->noise_seed = seed;
    h->noise_step = step;
    return CTCB_OK;
}

extern "C" int ctcb_brnn_set_zoneout(ctcb_brnn *h, float zc, float zh, uint64_t seed, const int64_t *step) {
    if (!h) return set_error(CTCB_EINVAL, "ctcb_brnn_set_zoneout: null handle");
    if (!(zc >= 0.f && zc < 1.f) || !(zh >= 0.f && zh < 1.f))
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_zoneout: zc = %g, zh = %g (need both in [0, 1))", (double)zc,
                         (double)zh);
    if ((zc > 0.f || zh > 0.f) && h->cfg.zoneout != 1)
        return set_error(CTCB_EINVAL, "ctcb_brnn_set_zoneout: zc = %g, zh = %g need zoneout = 1 in the config",
                         (double)zc, (double)zh);
    h->zo_c = zc;
    h->zo_h = zh;
    h->zo_seed = seed;
    h->zo_step = step;
    return CTCB_OK;
}

extern "C" int ctcb_brnn_weight_noise_f32(ctcb_brnn *h, const float *params, float *out, void *stream) {
    if (!h || !params || !out) return set_error(CTCB_EINVAL, "ctcb_brnn_weight_noise_f32: null pointer argument");
    const int64_t n = h->net.params;
    if (params < out + n && out < params + n)
        return set_error(CTCB_EINVAL, "ctcb_brnn_weight_noise_f32: out overlaps params");
    if (!h->noise_on()) {
        CTCB_CUDA_CHECK(cudaMemcpyAsync(out, params, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice,
                                        (cudaStream_t)stream));
        return CTCB_OK;
    }
    return run_weight_noise(params, out, n, h->noise_lo, h->noise_hi, h->noise_n, h->noise_sigma, h->noise_seed,
                            h->noise_step, (cudaStream_t)stream);
}

extern "C" size_t ctcb_brnn_sweep_workspace_bytes(int H, int B) { return 4096 + ctcb::sweep_tc_workspace_bytes(H, B); }

// ---- the step's reductions on their own: the same launches as the training call makes ---------------------------
extern "C" size_t ctcb_colsum_workspace_bytes(int64_t R, int n) {
    if (R <= 0 || n <= 0) return 0;
    return (size_t)((R + CS_ROWS_MIN - 1) / CS_ROWS_MIN) * (size_t)n * sizeof(float);
}

static int colsum_check(const char *fn, int64_t R, int n) {
    if (R <= 0 || n <= 0) return set_error(CTCB_EINVAL, "%s: R = %lld, n = %d (need R >= 1, n >= 1)", fn, (long long)R, n);
    if ((R + CS_ROWS_MIN - 1) / CS_ROWS_MIN > 65535)
        return set_error(CTCB_EINVAL, "%s: R = %lld rows exceed %d row blocks of %d", fn, (long long)R, 65535, CS_ROWS_MIN);
    return CTCB_OK;
}

extern "C" int ctcb_colsum_f32(const float *delta, int64_t R, int n, float *out, int accumulate, void *workspace,
                               size_t ws_bytes, void *stream) {
    if (int rc = colsum_check("ctcb_colsum_f32", R, n)) return rc;
    if (!delta || !out || !workspace) return set_error(CTCB_EINVAL, "ctcb_colsum_f32: null pointer argument");
    if (((uintptr_t)workspace) & 15) return set_error(CTCB_EINVAL, "ctcb_colsum_f32: workspace is not 16-byte aligned");
    const size_t need = ctcb_colsum_workspace_bytes(R, n);
    if (ws_bytes < need) return set_error(CTCB_ENOMEM, "ctcb_colsum_f32: workspace %zu < %zu bytes", ws_bytes, need);
    return run_colsum(delta, R, n, (float *)workspace, out, accumulate != 0, (cudaStream_t)stream);
}

extern "C" int ctcb_debug_colsum_plan(int64_t R, int n, const float *delta, int32_t *out) {
    if (int rc = colsum_check("ctcb_debug_colsum_plan", R, n)) return rc;
    if (!out) return set_error(CTCB_EINVAL, "ctcb_debug_colsum_plan: null pointer argument");
    const ColsumPlan p = colsum_plan(delta, R, n);
    out[0] = p.wide ? 1 : 0;
    out[1] = p.ncb;
    out[2] = (int32_t)p.rpb;
    out[3] = p.nblk;
    return CTCB_OK;
}

extern "C" int ctcb_softmax_rows_f32(const float *x, float *p, int64_t R, int K, void *stream) {
    if (!x || !p) return set_error(CTCB_EINVAL, "ctcb_softmax_rows_f32: null pointer argument");
    if (R <= 0 || K <= 0 || (R + 7) / 8 > 0x7fffffff)
        return set_error(CTCB_EINVAL, "ctcb_softmax_rows_f32: R = %lld, K = %d (need 1 <= R < 2^34, K >= 1)", (long long)R, K);
    return run_softmax_rows(x, p, R, K, (cudaStream_t)stream);
}

extern "C" int ctcb_softmax_rows_backward_f32(const float *p, const float *dp, const float *add, float *out, int64_t R,
                                              int K, void *stream) {
    if (!p || !dp || !out) return set_error(CTCB_EINVAL, "ctcb_softmax_rows_backward_f32: null pointer argument");
    if (R <= 0 || K <= 0 || (R + 7) / 8 > 0x7fffffff)
        return set_error(CTCB_EINVAL, "ctcb_softmax_rows_backward_f32: R = %lld, K = %d (need 1 <= R < 2^34, K >= 1)",
                         (long long)R, K);
    return run_softmax_rows_backward(p, dp, add, out, R, K, (cudaStream_t)stream);
}

// Test / diagnostic hook: where, inside the workspace, the activations of the LAST ctcb_brnn_cost_and_grad call lie
// (time-major [Tmax][B][n] with that call's B and Tmax).  what = 0: output of affine map `layer` (1..numLayers+1; the
// temporal layer's entry holds For + Back, the last one the logits), 1: For, 2: Back (temporal layer only; with
// several, `layer` says which, and only a bi-directional stack has a Back of every layer).  Subsampled nets: entries of
// maps >= L are [Tmax'][B][n]; what = 6: S, the stacked input of map L, k n wide.  what = 7: the delta of map `layer`,
// the buffer its weight and bias gradients read (Step::delta), where no later stage of the call overwrites it.
// what = 8..11 (interLayer > 0): the intermediate logits A, D_aux, the intermediate nll and skips.  what = 12..14
// (selfCondition = 1): X'_m, P, dA.  what = 15..17 (layer-normalised layer `layer`): z, Mu, Rstd.  what = 18
// (maskFeatDim > 0): the masked feature copy; 19 (weightNoise = 1): the noisy parameter copy.
extern "C" int ctcb_brnn_activation_offset(const ctcb_brnn_config *cfg, int what, int layer, size_t *offset, int32_t *width) {
    if (!valid_cfg(cfg) || !offset) return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: bad arguments");
    const WsLayout w = ws_layout(cfg);
    if (what >= 8 && what <= 11) {     // the intermediate CTC loss: A, D_aux, nll, skips
        if (cfg->interLayer <= 0)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: nothing of kind %d without interLayer", what);
        const size_t at[4] = {w.inter_A, w.inter_D, w.inter_nll, w.inter_skip};
        *offset = at[what - 8];
        if (width) *width = what <= 9 ? cfg->outputDim : 1;
        return CTCB_OK;
    }
    if (what >= 12 && what <= 14) {     // self-conditioned CTC: X'_m, P, dA
        if (cfg->selfCondition != 1)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: nothing of kind %d without selfCondition", what);
        const size_t at[3] = {w.cond_X, w.cond_P, w.cond_dA};
        *offset = at[what - 12];
        if (width) *width = what == 12 ? cfg->layerSize : cfg->outputDim;
        return CTCB_OK;
    }
    if (what >= 15 && what <= 17) {     // a layer-normalised layer: z, Mu, Rstd
        if (layer < 1 || layer > cfg->numLayers || !is_normed(cfg, layer))
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d is not layer-normalised", layer);
        const size_t at[3] = {w.Z[layer], w.Mu[layer], w.Rstd[layer]};
        *offset = at[what - 15];
        if (width) *width = what == 15 ? cfg->layerSize : 1;
        return CTCB_OK;
    }
    if (what == 18) {     // the masked copy of the features, [Tmax][B][inputDim]
        if (cfg->maskFeatDim <= 0)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: no masked feature copy without maskFeatDim");
        *offset = w.masked;
        if (width) *width = cfg->inputDim;
        return CTCB_OK;
    }
    if (what == 19) {     // the noisy copy of the flat parameter vector
        if (cfg->weightNoise != 1)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: no noisy parameter copy without weightNoise");
        *offset = w.noisy;
        if (width) *width = (int32_t)ctcb_brnn_param_count(cfg);
        return CTCB_OK;
    }
    if (what == 7) {
        if (layer < 1 || layer > cfg->numLayers + 1)
            return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d", layer);
        const int j = layer - eff_tl(cfg);
        if (cfg->unidirectional && cfg->cell != 1 && is_temporal(cfg, layer)) {
            // the BPTT result is the delta; layer j - 2 of the stack writes the same pair after it
            if (j >= 2)
                return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: the delta of map %d is overwritten by the "
                                 "call", layer);
            *offset = w.dFor[j % 2];
        } else {
            *offset = w.D[layer];
        }
        if (width) *width = map_rows(cfg, layer);
        return CTCB_OK;
    }
    if (what == 6 && eff_k(cfg) > 1) {
        *offset = w.S;
        if (width) *width = map_cols(cfg, cfg->subsampleLayer);
        return CTCB_OK;
    }
    if (what == 0) {
        if (layer < 1 || layer > cfg->numLayers + 1) return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d", layer);
        *offset = w.X[layer];
        if (width) *width = map_rows(cfg, layer);     // an LSTM layer's X holds its gates
        return CTCB_OK;
    }
    const int nt = eff_nt(cfg), tl = eff_tl(cfg);
    const bool lstm_kind = (what >= 3 && what <= 5);
    if ((what != 1 && what != 2 && !lstm_kind) || nt == 0 || (what == 2 && nt > 1 && cfg->unidirectional) ||
        (lstm_kind && cfg->cell != 1) || (what == 5 && cfg->unidirectional))
        return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: nothing of kind %d in this net", what);
    const int j = (nt == 1) ? 0 : layer - tl;     // one temporal layer: `layer` is ignored
    if (j < 0 || j >= nt)
        return set_error(CTCB_EINVAL, "ctcb_brnn_activation_offset: layer %d is not one of the temporal layers %d..%d",
                         layer, tl, tl + nt - 1);
    *offset = (what == 1) ? w.For[j] : (what == 2) ? w.Back[j] : (what == 3) ? w.X[tl + j] : (what == 4) ? w.Cf[j] : w.Cb[j];
    if (width) *width = (what == 3) ? map_rows(cfg, tl + j) : cfg->layerSize;
    return CTCB_OK;
}
