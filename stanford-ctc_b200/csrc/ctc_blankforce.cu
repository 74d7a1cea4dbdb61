// ctc_blankforce.cu -- the blank-forced CTC loss/gradient of the reference as an option of the CTC path
// (ctc_fast/ctc-loss/ctc_fast_blankforce.pyx:13-113).
//
// Differences from ctc.cu (ctc_fast.pyx): the label sequence arrives WITH its blanks, so the trellis has
// L = len(seq) states, transitions s -> s and s -> s+1 only (:51-52, :73-74), one start state (:43) and one
// end state (:64), no [start,end) window -- every state enters the frame normaliser (:55-59), so the
// returned cost is the log of the total mass of all states at the last frame.  State 0 is propagated with
// the probability of ROW 0 (`params[s,t]`, :49), not of seq[0]; kept as is.
//
// One CTA per utterance, float64 state as in the reference.  Per frame one block-wide reduction gives the
// normaliser c; the un-normalised states are exchanged through shared memory and every reader divides by c
// itself, so the alpha pass costs one barrier per frame and the beta/gradient pass two.  The normalised
// alpha trellis (T x L doubles) is spilled to the workspace; the probabilities are written into grad_out
// first (softmax of the logits, float32 as brnnet.py:170 hands them over) and each row is replaced by its
// gradient when the beta pass reaches it.  Occupancies are summed as 2^40 fixed point (integer shared
// atomics: order-independent, run-to-run identical).
#include <math_constants.h>

#include "common.cuh"

namespace ctcb {

constexpr int BF_THREADS = 256;
constexpr int BF_WARPS = BF_THREADS / 32;
constexpr int BF_SPT = 4;                      // states per thread -> at most 1024 states
constexpr double BF_FIX = 1099511627776.0;     // 2^40

struct BfArgs {
    const float *acts;
    int is_prob;
    int64_t us, fs;
    const int32_t *seq, *soff, *Tlen;
    int B, Tmax, K, Lmax;
    float *grad, *nll;
    int32_t *skip;
    double *ws;
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum over the CTA; `slot` is a [BF_WARPS] shared array that the caller alternates between consecutive calls,
// so one barrier per reduction is enough.  Fixed summation order: the result is identical in every thread.
__device__ __forceinline__ double block_sum(double v, double *slot) {
    v = warp_sum_d(v);
    if ((threadIdx.x & 31) == 0) slot[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < BF_WARPS; ++w) s += slot[w];
    return s;
}

__global__ void __launch_bounds__(BF_THREADS) ctc_blankforce_kernel(BfArgs a) {
    extern __shared__ double sm_d[];
    const int u = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = a.K;
    const int T = min(a.Tlen[u], a.Tmax);
    const int so = a.soff[u];
    const int L = a.soff[u + 1] - so;
    const int Lp = a.Lmax;
    double *xbuf = sm_d;                                  // [2][Lp] un-normalised states of two frames
    double *red = xbuf + 2 * Lp;                          // [2][2][BF_WARPS]
    unsigned long long *occ = (unsigned long long *)(red + 4 * BF_WARPS);   // [K]
    int *lab = (int *)(occ + K);                          // [Lp]
    const float *acts = a.acts + (int64_t)u * a.us;
    float *g = a.grad + (int64_t)u * a.us;
    double *trellis = a.ws + (int64_t)u * a.Tmax * Lp;

    // ---- probabilities into grad_out (rows >= T: zero gradient)
    for (int t = warp; t < a.Tmax; t += BF_WARPS) {
        const float *xr = acts + (int64_t)t * a.fs;
        float *pr = g + (int64_t)t * a.fs;
        if (t >= T) {
            for (int k = lane; k < K; k += 32) pr[k] = 0.f;
        } else if (a.is_prob) {
            for (int k = lane; k < K; k += 32) pr[k] = xr[k];
        } else {                                           // brnnet.py:161-168, float32
            float m = -3.4e38f;
            for (int k = lane; k < K; k += 32) m = fmaxf(m, xr[k]);
            m = warp_max(m);
            float z = 0.f;
            for (int k = lane; k < K; k += 32) z += expf(xr[k] - m);
            z = warp_sum(z);
            const float inv = 1.f / z;
            for (int k = lane; k < K; k += 32) pr[k] = expf(xr[k] - m) * inv;
        }
    }
    for (int s = tid; s < L; s += BF_THREADS) lab[s] = a.seq[so + s];
    for (int k = tid; k < K; k += BF_THREADS) occ[k] = 0ull;
    if (T <= 0 || L <= 0 || L > BF_SPT * BF_THREADS) {     // nothing the reference could evaluate
        if (tid == 0) { a.nll[u] = 0.f; a.skip[u] = 1; }
        return;
    }
    __syncthreads();

    int myl[BF_SPT];
#pragma unroll
    for (int j = 0; j < BF_SPT; ++j) {
        const int s = tid + j * BF_THREADS;
        myl[j] = (s < L) ? lab[s] : 0;
    }
    // row of the probability each state multiplies with in the ALPHA pass: state 0 uses row 0 (:49)
    auto alpha_row = [&](int j) { return (tid + j * BF_THREADS == 0) ? 0 : myl[j]; };

    bool fail = false;
    // ------------------------------------------------------------------ alpha (:43-59)
    double llF = log((double)g[lab[0]]);                   // :44, frame 0
    double c_prev = 1.0;
#pragma unroll
    for (int j = 0; j < BF_SPT; ++j) {
        const int s = tid + j * BF_THREADS;
        if (s < L) xbuf[s] = (s == 0) ? 1.0 : 0.0;          // :43
    }
    __syncthreads();
    float pn[BF_SPT];
#pragma unroll
    for (int j = 0; j < BF_SPT; ++j) pn[j] = (T > 1 && tid + j * BF_THREADS < L) ? g[a.fs + alpha_row(j)] : 0.f;
    for (int t = 1; t < T; ++t) {
        const double *xp = xbuf + ((t - 1) & 1) * Lp;
        double *xc = xbuf + (t & 1) * Lp;
        float pc[BF_SPT];
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            pc[j] = pn[j];
            pn[j] = (t + 1 < T && tid + j * BF_THREADS < L) ? g[(int64_t)(t + 1) * a.fs + alpha_row(j)] : 0.f;
        }
        double part = 0.0;
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            const int s = tid + j * BF_THREADS;
            if (s < L) {
                const double ap = xp[s] / c_prev;                         // normalised alpha[s, t-1] (:57-58)
                trellis[(int64_t)(t - 1) * Lp + s] = ap;
                const double am = (s > 0) ? xp[s - 1] / c_prev : 0.0;
                const double v = (s == 0) ? ap * (double)pc[j] : (ap + am) * (double)pc[j];   // :48-52
                xc[s] = v;
                part += v;
            }
        }
        const double c = block_sum(part, red + (t & 1) * BF_WARPS);
        if (c == 0.0) { fail = true; break; }               // ZeroDivisionError in the reference (:108)
        llF += log(c);
        c_prev = c;
    }
    if (!fail) {
        const double *xp = xbuf + ((T - 1) & 1) * Lp;
        for (int s = tid; s < L; s += BF_THREADS) trellis[(int64_t)(T - 1) * Lp + s] = xp[s] / c_prev;
    }
    __syncthreads();

    // ------------------------------------------------------------------ beta + gradient (:62-106)
    if (!fail) {
        double *red2 = red + 2 * BF_WARPS;
        c_prev = 1.0;
        float bn[BF_SPT];
        double an[BF_SPT];
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            const int s = tid + j * BF_THREADS;
            bn[j] = (s < L) ? g[(int64_t)(T - 1) * a.fs + myl[j]] : 0.f;
            an[j] = (s < L) ? trellis[(int64_t)(T - 1) * Lp + s] : 0.0;
        }
        for (int t = T - 1; t >= 0; --t) {
            const int step = T - 1 - t;
            const double *xp = xbuf + ((step + 1) & 1) * Lp;
            double *xc = xbuf + (step & 1) * Lp;
            float pc[BF_SPT];
            double al[BF_SPT];
#pragma unroll
            for (int j = 0; j < BF_SPT; ++j) {
                const int s = tid + j * BF_THREADS;
                pc[j] = bn[j];
                al[j] = an[j];
                bn[j] = (t > 0 && s < L) ? g[(int64_t)(t - 1) * a.fs + myl[j]] : 0.f;
                an[j] = (t > 0 && s < L) ? trellis[(int64_t)(t - 1) * Lp + s] : 0.0;
            }
            double w[BF_SPT];
            double part_c = 0.0, part_q = 0.0;
#pragma unroll
            for (int j = 0; j < BF_SPT; ++j) {
                const int s = tid + j * BF_THREADS;
                w[j] = 0.0;
                if (s < L) {
                    double v;
                    if (t == T - 1) {
                        v = (s == L - 1) ? 1.0 : 0.0;                                   // :64
                    } else {
                        const double bp = xp[s] / c_prev;
                        const double bq = (s < L - 1) ? xp[s + 1] / c_prev : 0.0;
                        v = (s == L - 1) ? bp * (double)pc[j] : (bp + bq) * (double)pc[j];   // :71-74
                    }
                    xc[s] = v;
                    part_c += v;
                    // alpha*beta/p of :85-92, still carrying the factor c of this frame
                    const double ab = al[j] * v;
                    if (ab != 0.0 && pc[j] != 0.f) w[j] = ab / (double)pc[j];
                    part_q += w[j];
                }
            }
            // both sums with one barrier
            part_c = warp_sum_d(part_c);
            part_q = warp_sum_d(part_q);
            double *slot = ((step & 1) ? red2 : red);
            if (lane == 0) { slot[warp] = part_c; slot[BF_WARPS + warp] = part_q; }
            __syncthreads();
            double c = 0.0, q = 0.0;
#pragma unroll
            for (int x = 0; x < BF_WARPS; ++x) { c += slot[x]; q += slot[BF_WARPS + x]; }
            if (c == 0.0) { fail = true; break; }
            c_prev = c;
            if (q > 0.0) {
#pragma unroll
                for (int j = 0; j < BF_SPT; ++j)
                    if (w[j] != 0.0)
                        atomicAdd(&occ[myl[j]], (unsigned long long)(w[j] / q * BF_FIX + 0.5));
            }
            __syncthreads();
            const double absum = q / c;                                                   // :94-97
            float *pr = g + (int64_t)t * a.fs;
            for (int k = tid; k < K; k += BF_THREADS) {
                const double p = (double)pr[k];
                const double tmp = p * absum;                                             // :102
                const double gam = (double)occ[k] * (1.0 / BF_FIX);
                occ[k] = 0ull;
                pr[k] = (float)((tmp > 0.0) ? p - gam : p);                               // :103-106
            }
        }
    }
    __syncthreads();
    if (fail) {                                            // skipped utterances carry no gradient
        for (int t = warp; t < T; t += BF_WARPS)
            for (int k = lane; k < K; k += 32) g[(int64_t)t * a.fs + k] = 0.f;
    }
    if (tid == 0) { a.nll[u] = (float)(-llF); a.skip[u] = fail ? 1 : 0; }
}

static size_t bf_smem(int K, int Lmax) {
    return sizeof(double) * (2 * (size_t)Lmax + 4 * BF_WARPS) + sizeof(unsigned long long) * (size_t)K + sizeof(int) * (size_t)Lmax;
}

}  // namespace ctcb

using namespace ctcb;

extern "C" size_t ctcb_ctc_blankforce_workspace_bytes(int B, int Tmax, int max_states) {
    if (B <= 0 || Tmax <= 0 || max_states <= 0 || max_states > BF_SPT * BF_THREADS) return 0;
    return (size_t)B * (size_t)Tmax * (size_t)max_states * sizeof(double);
}

extern "C" int ctcb_ctc_blankforce_loss_grad_f32(const float *acts, int is_prob, int64_t utt_stride,
                                                 int64_t frame_stride, const int32_t *seq, const int32_t *seq_off,
                                                 const int32_t *T_per_utt, int B, int Tmax, int K, int max_states,
                                                 float *grad_out, float *nll_out, int32_t *skip_out,
                                                 void *workspace, size_t ws_bytes, void *stream) {
    if (B <= 0) return CTCB_OK;
    if (!acts || !seq || !seq_off || !T_per_utt || !grad_out || !nll_out || !skip_out)
        return set_error(CTCB_EINVAL, "ctcb_ctc_blankforce_loss_grad_f32: null pointer argument");
    if (K <= 0 || Tmax <= 0)
        return set_error(CTCB_EINVAL, "ctcb_ctc_blankforce_loss_grad_f32: bad sizes K=%d Tmax=%d", K, Tmax);
    if (max_states <= 0 || max_states > BF_SPT * BF_THREADS)
        return set_error(CTCB_EINVAL, "ctcb_ctc_blankforce_loss_grad_f32: 1..%d states supported (got %d)",
                         BF_SPT * BF_THREADS, max_states);
    if (acts == grad_out)
        return set_error(CTCB_EINVAL, "ctcb_ctc_blankforce_loss_grad_f32: grad_out must not alias acts");
    const size_t need = ctcb_ctc_blankforce_workspace_bytes(B, Tmax, max_states);
    if (!workspace || ws_bytes < need)
        return set_error(CTCB_ENOMEM, "ctcb_ctc_blankforce_loss_grad_f32: workspace %zu < %zu bytes", ws_bytes, need);
    BfArgs a;
    a.acts = acts; a.is_prob = is_prob; a.us = utt_stride; a.fs = frame_stride;
    a.seq = seq; a.soff = seq_off; a.Tlen = T_per_utt;
    a.B = B; a.Tmax = Tmax; a.K = K; a.Lmax = max_states;
    a.grad = grad_out; a.nll = nll_out; a.skip = skip_out; a.ws = (double *)workspace;
    const size_t smem = bf_smem(K, max_states);
    if (smem > 200 * 1024)
        return set_error(CTCB_EINVAL, "ctcb_ctc_blankforce_loss_grad_f32: K=%d too large for shared memory", K);
    CTCB_CUDA_CHECK(cudaFuncSetAttribute(ctc_blankforce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ctc_blankforce_kernel<<<B, BF_THREADS, smem, (cudaStream_t)stream>>>(a);
    CTCB_LAUNCH_CHECK();
    return CTCB_OK;
}
