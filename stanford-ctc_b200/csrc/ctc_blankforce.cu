// ctc_blankforce.cu -- the blank-forced CTC loss/gradient of the reference as an option of the CTC path
// (ctc_fast/ctc-loss/ctc_fast_blankforce.pyx:13-113).
//
// Differences from ctc.cu (ctc_fast.pyx): the label sequence arrives WITH its blanks, so the trellis has
// L = len(seq) states, transitions s -> s and s -> s+1 only (:51-52, :73-74), one start state (:43) and one
// end state (:64), no [start,end) window -- every state enters the frame normaliser (:55-59), so the
// returned cost is the log of the total mass of all states at the last frame.  State 0 is propagated with
// the probability of ROW 0 (`params[s,t]`, :49), not of seq[s]; kept as is.
//
// One CTA per utterance, float64 state.  Unlike the reference, both passes run in the log domain with no per-frame
// normalisation: the reference's normalised alpha and beta and their product underflow float64 on long utterances
// with unaligned outputs (gradient rows left at p from ~3000 frames x 600 states, a loss off by hundreds of nats
// further out).  Here log alpha and log beta have the range of float64's exponent, and an occupancy is
// exp(la + lb - log p - frame max) / sum, which cannot underflow where it matters.  "A normaliser is 0" becomes "every
// state is -inf", so the reference's skips stay exact.  The alpha pass exchanges neighbouring states through shared
// memory (one barrier per frame); the beta/gradient pass needs a block reduction of (max, sum) pairs and the
// occupancy atomics (two barriers).  log alpha (T x L doubles) is spilled to the workspace; the probabilities are
// written into grad_out first (softmax of the logits, float32 as brnnet.py:170 hands them over) and each row is
// replaced by its gradient when the beta pass reaches it.  Occupancies are summed as 2^40 fixed point (integer shared
// atomics: order-independent, run-to-run identical).
//
// An utterance with no frame, no state, more states than max_states or a label outside [0, K) is skipped with a zero
// gradient; the check comes before anything reads its states.
#include <math_constants.h>

#include "common.cuh"

namespace ctcb {

constexpr int BF_THREADS = 256;
constexpr int BF_WARPS = BF_THREADS / 32;
constexpr int BF_SPT = 4;                      // states per thread -> at most 1024 states
constexpr double BF_FIX = 1099511627776.0;     // 2^40
constexpr double NEG_INF = -__builtin_huge_val();

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

__device__ __forceinline__ double lse2(double a, double b) {
    const double m = fmax(a, b);
    if (m == NEG_INF) return m;
    return m + log1p(exp(-fabs(a - b)));
}

// (m, s) stands for s * e^m.  Symmetric in its two operands bit for bit, so both lanes of a shuffle get the same pair.
__device__ __forceinline__ void ms_add(double &m, double &s, double om, double os) {
    const double n = fmax(m, om);
    if (n == NEG_INF) return;
    s = s * exp(m - n) + os * exp(om - n);
    m = n;
}

__device__ __forceinline__ void warp_ms(double &m, double &s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ms_add(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
}

// Combine the warps' pairs of `slot` ([2][BF_WARPS]) in a fixed order: the result is identical in every thread.
__device__ __forceinline__ void block_ms(const double *slot, double &m, double &s) {
    m = NEG_INF;
    s = 0.0;
#pragma unroll
    for (int w = 0; w < BF_WARPS; ++w) ms_add(m, s, slot[w], slot[BF_WARPS + w]);
}

__global__ void __launch_bounds__(BF_THREADS) ctc_blankforce_kernel(BfArgs a) {
    extern __shared__ double sm_d[];
    const int u = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = a.K;
    const int T = min(a.Tlen[u], a.Tmax);
    const int so = a.soff[u];
    const int L = a.soff[u + 1] - so;
    const int Lp = a.Lmax;
    double *xbuf = sm_d;                                  // [2][Lp] log states of two frames
    double *red = xbuf + 2 * Lp;                          // [2][2][BF_WARPS] (max, sum) pairs
    unsigned long long *occ = (unsigned long long *)(red + 4 * BF_WARPS);   // [K]
    int *lab = (int *)(occ + K);                          // [Lp]
    const float *acts = a.acts + (int64_t)u * a.us;
    float *g = a.grad + (int64_t)u * a.us;
    double *trellis = a.ws + (int64_t)u * a.Tmax * Lp;

    // ---- what the reference could not evaluate, or would read out of bounds for: skip with a zero gradient
    bool bad = T <= 0 || L <= 0 || L > Lp;
    if (!bad)
        for (int s = tid; s < L; s += BF_THREADS) {
            const int l = a.seq[so + s];
            if (l < 0 || l >= K) bad = true;
            else lab[s] = l;
        }
    bad = __syncthreads_or(bad);

    // ---- probabilities into grad_out (rows >= T, and every row of a skipped utterance: zero gradient)
    for (int t = warp; t < a.Tmax; t += BF_WARPS) {
        const float *xr = acts + (int64_t)t * a.fs;
        float *pr = g + (int64_t)t * a.fs;
        if (t >= T || bad) {
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
    if (bad) {
        if (tid == 0) { a.nll[u] = 0.f; a.skip[u] = 1; }
        return;
    }
    for (int k = tid; k < K; k += BF_THREADS) occ[k] = 0ull;
    __syncthreads();

    int myl[BF_SPT];
#pragma unroll
    for (int j = 0; j < BF_SPT; ++j) {
        const int s = tid + j * BF_THREADS;
        myl[j] = (s < L) ? lab[s] : 0;
    }
    // row of the probability each state multiplies with in the ALPHA pass: state 0 uses row 0 (:49)
    auto alpha_row = [&](int j) { return (tid + j * BF_THREADS == 0) ? 0 : myl[j]; };

    // ------------------------------------------------------------------ log alpha (:43-59)
    double la[BF_SPT];
#pragma unroll
    for (int j = 0; j < BF_SPT; ++j) {
        const int s = tid + j * BF_THREADS;
        la[j] = (s == 0) ? 0.0 : NEG_INF;                  // alpha(0,0) = 1, no emission (:43)
        if (s < L) xbuf[s] = la[j];
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
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            const int s = tid + j * BF_THREADS;
            if (s < L) {
                trellis[(int64_t)(t - 1) * Lp + s] = la[j];
                const double v = (s == 0) ? la[j] : lse2(la[j], xp[s - 1]);            // :48-52
                la[j] = v + log((double)pc[j]);
                xc[s] = la[j];
            }
        }
        __syncthreads();
    }
    // -llForward = -(log p[seq[0],0] + log of the mass of all states at T-1) (:44, :55-59)
    double *red2 = red + 2 * BF_WARPS;
    double llF, logZ;
    {
        double m = NEG_INF, sm = 0.0;
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            const int s = tid + j * BF_THREADS;
            if (s < L) {
                trellis[(int64_t)(T - 1) * Lp + s] = la[j];
                ms_add(m, sm, la[j], 1.0);
            }
        }
        warp_ms(m, sm);
        if (lane == 0) { red2[warp] = m; red2[BF_WARPS + warp] = sm; }
        __syncthreads();
        block_ms(red2, m, sm);
        logZ = (m == NEG_INF) ? NEG_INF : m + log(sm);
        llF = log((double)g[lab[0]]) + logZ;
    }
    // the mass of the last frame is 0 exactly when a frame normaliser of the reference is (:108)
    bool fail = logZ == NEG_INF;
    bool zero_p = false;

    // ------------------------------------------------------------------ log beta + gradient (:62-106)
    if (!fail) {
        double lb[BF_SPT];
        float bn[BF_SPT];
        double an[BF_SPT];
#pragma unroll
        for (int j = 0; j < BF_SPT; ++j) {
            const int s = tid + j * BF_THREADS;
            lb[j] = NEG_INF;
            bn[j] = (s < L) ? g[(int64_t)(T - 1) * a.fs + myl[j]] : 0.f;
            an[j] = (s < L) ? trellis[(int64_t)(T - 1) * Lp + s] : NEG_INF;
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
                an[j] = (t > 0 && s < L) ? trellis[(int64_t)(t - 1) * Lp + s] : NEG_INF;
            }
            double e[BF_SPT];
            double m = NEG_INF, sm = 0.0;
            bool alive = false;
#pragma unroll
            for (int j = 0; j < BF_SPT; ++j) {
                const int s = tid + j * BF_THREADS;
                e[j] = NEG_INF;
                if (s < L) {
                    const double lpk = log((double)pc[j]);
                    double v;
                    if (t == T - 1) v = (s == L - 1) ? 0.0 : NEG_INF;                           // :64
                    else v = ((s == L - 1) ? lb[j] : lse2(lb[j], xp[s + 1])) + lpk;              // :71-74
                    lb[j] = v;
                    xc[s] = v;
                    alive |= v != NEG_INF;
                    // alpha*beta/p of :85-92; alpha*beta != 0 where p == 0 is the reference's skip (:88-92)
                    const double ab = al[j] + v;
                    if (ab != NEG_INF) {
                        if (pc[j] == 0.f) {
                            zero_p = true;
                        } else {
                            e[j] = ab - lpk;
                            ms_add(m, sm, e[j], 1.0);
                        }
                    }
                }
            }
            warp_ms(m, sm);
            double *slot = ((step & 1) ? red2 : red);
            if (lane == 0) { slot[warp] = m; slot[BF_WARPS + warp] = sm; }
            if (!__syncthreads_or(alive)) { fail = true; break; }                  // beta normaliser 0 (:108)
            block_ms(slot, m, sm);
            const bool any = m != NEG_INF;                                         // absum > 0 (:94-97)
            if (any) {
#pragma unroll
                for (int j = 0; j < BF_SPT; ++j)
                    if (e[j] != NEG_INF)
                        atomicAdd(&occ[myl[j]], (unsigned long long)(exp(e[j] - m) / sm * BF_FIX + 0.5));
            }
            __syncthreads();
            float *pr = g + (int64_t)t * a.fs;
            for (int k = tid; k < K; k += BF_THREADS) {
                const double p = (double)pr[k];
                const double gam = (double)occ[k] * (1.0 / BF_FIX);
                occ[k] = 0ull;
                pr[k] = (float)((any && p > 0.0) ? p - gam : p);                   // tmp > 0 rule (:102-106)
            }
        }
    }
    fail = __syncthreads_or(fail || zero_p);
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
