/*
 * oracle/ctc_oracle.c -- TEST INFRASTRUCTURE ONLY (checker + CPU baseline "port").
 *
 * Plain-C float64 restatement of the reference CTC forward-backward,
 *   ctc_fast/ctc-loss/ctc_fast.pyx:13-152  (ctc_loss)
 *   ctc_fast/ctc-loss/ctc_fast.pyx:154-187 (decode_best_path)
 * Parity pinned: validated against the unmodified .pyx compiled into oracle/_ref/
 * (tests/test_oracle.py) and the known-answer value of ctc/time_trials.py:13-25
 * (NLL 1710.233966660).  Never linked or called by the product library.
 *
 * params is K x T in Fortran order (frame-contiguous: params[k + K*t]), as the reference
 * requires (ctc_fast.pyx:13).  Returns skip (0/1); *nll receives -llForward.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define P(k, t) params[(size_t)(k) + (size_t)K * (size_t)(t)]
#define A(s, t) alphas[(size_t)(s) + (size_t)L * (size_t)(t)]
#define B(s, t) betas[(size_t)(s) + (size_t)L * (size_t)(t)]
#define AB(s, t) ab[(size_t)(s) + (size_t)L * (size_t)(t)]
#define G(k, t) grad[(size_t)(k) + (size_t)K * (size_t)(t)]

/* *llb, when not NULL, receives the llBackward the reference computes and discards (:84-114).  With exact
 * arithmetic it equals llForward; where the per-frame normalised trellis loses mass to float64 underflow the two
 * disagree. */
int ctc_oracle_loss_fb(const double *params, int K, int T, const int *seq, int seqLen,
                       int blank, double *grad, double *nll, double *llb)
{
    /* ctc_fast.pyx:23-34 -- sizes and zero-initialised trellises */
    int L = 2 * seqLen + 1;
    double *alphas = (double *)calloc((size_t)L * T, sizeof(double));
    double *betas = (double *)calloc((size_t)L * T, sizeof(double));
    double *ab = (double *)malloc((size_t)L * T * sizeof(double));
    double *absum = (double *)malloc((size_t)T * sizeof(double));
    double c, llForward = 0.0, llBackward = 0.0, tmp;
    int t, s, l, start, end, skip = 0;
    memset(grad, 0, (size_t)K * T * sizeof(double));

    /* ctc_fast.pyx:42-47 -- alpha init.  A zero normaliser raises ZeroDivisionError in the
     * reference (Cython checked division) which it turns into skip=True (:147-149). */
    A(0, 0) = P(blank, 0);
    A(1, 0) = P(seq[0], 0);
    c = A(0, 0) + A(1, 0);
    if (c == 0.0) { skip = 1; goto done; }
    A(0, 0) /= c;
    A(1, 0) /= c;
    llForward = log(c);
    for (t = 1; t < T; t++) {
        /* :49-54 -- window of states that can still reach the end / be reached */
        start = 2 * (T - t);
        start = (L <= start) ? 0 : L - start;
        end = (2 * t + 2 < L) ? 2 * t + 2 : L;
        for (s = start; s < L; s++) {            /* :55-68 */
            l = (s - 1) / 2;
            if (s % 2 == 0) {
                if (s == 0) A(s, t) = A(s, t - 1) * P(blank, t);
                else A(s, t) = (A(s, t - 1) + A(s - 1, t - 1)) * P(blank, t);
            } else if (s == 1 || seq[l] == seq[l - 1]) {
                A(s, t) = (A(s, t - 1) + A(s - 1, t - 1)) * P(seq[l], t);
            } else {
                A(s, t) = (A(s, t - 1) + A(s - 1, t - 1) + A(s - 2, t - 1)) * P(seq[l], t);
            }
        }
        c = 0.0;                                  /* :70-76 */
        for (s = start; s < end; s++) c += A(s, t);
        if (c == 0.0 && start < end) { skip = 1; goto done; }
        for (s = start; s < end; s++) A(s, t) /= c;
        llForward += log(c);                      /* empty window: log(0) = -inf, no raise */
    }

    /* :78-83 -- beta init */
    B(L - 1, T - 1) = P(blank, T - 1);
    B(L - 2, T - 1) = P(seq[seqLen - 1], T - 1);
    c = B(L - 1, T - 1) + B(L - 2, T - 1);
    if (c == 0.0) { skip = 1; goto done; }
    B(L - 1, T - 1) /= c;
    B(L - 2, T - 1) /= c;
    llBackward = log(c);
    for (t = T - 2; t >= 0; t--) {                /* :84-114 */
        start = 2 * (T - t);
        start = (L <= start) ? 0 : L - start;
        end = (2 * t + 2 < L) ? 2 * t + 2 : L;
        for (s = end - 1; s >= 0; s--) {
            l = (s - 1) / 2;
            if (s % 2 == 0) {
                if (s == L - 1) B(s, t) = B(s, t + 1) * P(blank, t);
                else B(s, t) = (B(s, t + 1) + B(s + 1, t + 1)) * P(blank, t);
            } else if (s == L - 2 || seq[l] == seq[l + 1]) {
                B(s, t) = (B(s, t + 1) + B(s + 1, t + 1)) * P(seq[l], t);
            } else {
                B(s, t) = (B(s, t + 1) + B(s + 1, t + 1) + B(s + 2, t + 1)) * P(seq[l], t);
            }
        }
        c = 0.0;
        for (s = start; s < end; s++) c += B(s, t);
        if (c == 0.0 && start < end) { skip = 1; goto done; }
        for (s = start; s < end; s++) B(s, t) /= c;
        llBackward += log(c);
    }

    /* :117-131 -- posterior occupancy numerators and the ab/p trellis */
    for (t = 0; t < T; t++)
        for (s = 0; s < L; s++) AB(s, t) = A(s, t) * B(s, t);
    for (s = 0; s < L; s++) {
        int k = (s % 2 == 0) ? blank : seq[(s - 1) / 2];
        for (t = 0; t < T; t++) {
            G(k, t) += AB(s, t);
            if (AB(s, t) != 0) AB(s, t) = AB(s, t) / P(k, t);
        }
    }
    for (t = 0; t < T; t++) {                     /* :133-136 */
        absum[t] = 0;
        for (s = 0; s < L; s++) absum[t] += AB(s, t);
    }
    for (t = 0; t < T; t++)                       /* :139-145 */
        for (s = 0; s < K; s++) {
            tmp = P(s, t) * absum[t];
            if (tmp > 0) G(s, t) = P(s, t) - G(s, t) / tmp;
            else G(s, t) = P(s, t);
        }

done:
    /* on skip the reference returns grad as accumulated so far: still all zeros */
    *nll = -llForward;
    if (llb) *llb = llBackward;
    free(alphas); free(betas); free(ab); free(absum);
    return skip;
}

int ctc_oracle_loss(const double *params, int K, int T, const int *seq, int seqLen,
                    int blank, double *grad, double *nll)
{
    return ctc_oracle_loss_fb(params, K, T, seq, seqLen, blank, grad, nll, NULL);
}

/*
 * The same loss and gradient in the log domain: float64 log-sum-exp recursions with no per-frame scaling, so no
 * state and no product of alpha and beta leaves float64's range however long the utterance.  Where the scaled
 * restatement above is in range the two agree to rounding; where it is not (thousands of frames, unaligned
 * outputs) this one is the truth the tests hold the kernel to.  The reference's contract is kept:
 *   T < |l|            -> (inf, grad = p, no skip); a one-frame utterance returns -log(p[blank,0] + p[l_0,0]),
 *                         as the reference's un-windowed initialisation does (:42-47), and skips when that is 0;
 *   no alignment (P=0) -> skip with a zero gradient (the reference's ZeroDivisionError, :147-149).
 * g = p - gamma, gamma[k,t] = sum over states s of label k of exp(la[s,t] + lb[s,t] - log p[k,t] - log P).
 */
static double lse2(double a, double b)
{
    double m = a > b ? a : b;
    if (m == -INFINITY) return -INFINITY;
    return m + log(exp(a - m) + exp(b - m));
}

static double lse3(double a, double b, double c)
{
    double m = a > b ? a : b;
    m = m > c ? m : c;
    if (m == -INFINITY) return -INFINITY;
    return m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

int ctc_oracle_loss_log(const double *params, int K, int T, const int *seq, int seqLen,
                        int blank, double *grad, double *nll)
{
    int L = 2 * seqLen + 1, t, s, k;
    int *lab = (int *)malloc((size_t)L * sizeof(int));
    double *la, *lb, *lp, logP;
    memset(grad, 0, (size_t)K * T * sizeof(double));
    for (s = 0; s < L; s++) lab[s] = (s % 2 == 0) ? blank : seq[(s - 1) / 2];

    if (T == 1) {                                      /* the reference's normaliser of frame 0 */
        double c = P(blank, 0) + P(seq[0], 0);
        if (c == 0.0) { *nll = -log(c); free(lab); return 1; }
        *nll = -log(c);
    } else if (T < seqLen) {
        *nll = INFINITY;
    }
    if (T < seqLen) {
        for (t = 0; t < T; t++)
            for (k = 0; k < K; k++) G(k, t) = P(k, t);
        free(lab);
        return 0;
    }

    la = (double *)malloc((size_t)L * T * sizeof(double));
    lb = (double *)malloc((size_t)L * T * sizeof(double));
    lp = (double *)malloc((size_t)K * T * sizeof(double));
    for (t = 0; t < T; t++)
        for (k = 0; k < K; k++) lp[(size_t)k + (size_t)K * t] = log(P(k, t));
#define LP(k, t) lp[(size_t)(k) + (size_t)K * (size_t)(t)]
#define LA(s, t) la[(size_t)(s) + (size_t)L * (size_t)(t)]
#define LB(s, t) lb[(size_t)(s) + (size_t)L * (size_t)(t)]
    for (s = 0; s < L; s++) LA(s, 0) = (s < 2) ? LP(lab[s], 0) : -INFINITY;
    for (t = 1; t < T; t++)
        for (s = 0; s < L; s++) {
            double x;
            if (s == 0) x = LA(0, t - 1);
            else if (s % 2 == 0 || s == 1 || lab[s] == lab[s - 2]) x = lse2(LA(s, t - 1), LA(s - 1, t - 1));
            else x = lse3(LA(s, t - 1), LA(s - 1, t - 1), LA(s - 2, t - 1));
            LA(s, t) = x + LP(lab[s], t);
        }
    for (s = 0; s < L; s++) LB(s, T - 1) = (s >= L - 2) ? LP(lab[s], T - 1) : -INFINITY;
    for (t = T - 2; t >= 0; t--)
        for (s = L - 1; s >= 0; s--) {
            double x;
            if (s == L - 1) x = LB(s, t + 1);
            else if (s % 2 == 0 || s == L - 2 || lab[s] == lab[s + 2]) x = lse2(LB(s, t + 1), LB(s + 1, t + 1));
            else x = lse3(LB(s, t + 1), LB(s + 1, t + 1), LB(s + 2, t + 1));
            LB(s, t) = x + LP(lab[s], t);
        }
    logP = (L > 1) ? lse2(LA(L - 1, T - 1), LA(L - 2, T - 1)) : LA(0, T - 1);
    if (logP == -INFINITY) {
        free(la); free(lb); free(lp);
        free(lab);
        if (T == 1) {                                  /* the reference: absum == 0 leaves grad = p */
            for (k = 0; k < K; k++) G(k, 0) = P(k, 0);
            return 0;
        }
        *nll = INFINITY;                               /* no alignment: skip, gradient all zeros */
        return 1;
    }
    if (T > 1) *nll = -logP;
    for (t = 0; t < T; t++)
        for (s = 0; s < L; s++) {
            double e = LA(s, t) + LB(s, t);
            if (e != -INFINITY) G(lab[s], t) += exp(e - LP(lab[s], t) - logP);
        }
    for (t = 0; t < T; t++)
        for (k = 0; k < K; k++) G(k, t) = P(k, t) - G(k, t);
#undef LP
#undef LA
#undef LB
    free(lab); free(la); free(lb); free(lp);
    return 0;
}

/* The label np.argmax picks in frame t (ctc_fast.pyx:167, ctc_fast_blankforce.pyx:132): the first NaN if the frame has
 * one, else the first maximum; a frame of -inf gives 0. */
static int argmax_frame(const double *probs, int K, int t)
{
    const double *row = probs + (size_t)K * t;
    int b = 0, k;
    for (k = 1; k < K && !isnan(row[b]); k++)
        if (isnan(row[k]) || row[k] > row[b]) b = k;
    return b;
}

/* ctc_fast.pyx:154-187 -- per-frame argmax, collapse repeats, drop blank and labels 1,2,8.
 * hyp/align must hold T ints; returns the hypothesis length. */
int ctc_oracle_best_path(const double *probs, int K, int T, int blank, int *hyp, int *align)
{
    int n = 0, prev = -1, t;
    for (t = 0; t < T; t++) {
        int b = argmax_frame(probs, K, t);
        if (b == blank) { prev = b; continue; }                 /* :172-173 */
        if (b == 1 || b == 2 || b == 8) { prev = b; continue; } /* :176-177 */
        if (t != 0 && b == prev) { if (n > 0) align[n - 1] = t; prev = b; continue; } /* :179-181 */
        hyp[n] = b; align[n] = t; n++;
        prev = b;
    }
    return n;
}

/*
 * Blank-forced variant: ctc_fast/ctc-loss/ctc_fast_blankforce.pyx:13-113.
 * `seq` already contains the blanks (:24-26): L = seqLen states, transitions s -> s and s -> s+1
 * only (:51-52), a single start state (:43) and a single end state (:64); every state enters the
 * per-frame normaliser (:55-59), so -llForward is the log of the total mass of ALL states at T-1.
 * Quirk kept: state 0 is propagated with params[0,t] -- row index s, not seq[s] (:49).
 * Same skip rule: a zero normaliser raises ZeroDivisionError in the reference (:108-110).
 */
int ctc_oracle_loss_blankforce(const double *params, int K, int T, const int *seq, int seqLen,
                               double *grad, double *nll)
{
    int L = seqLen;
    double *alphas = (double *)calloc((size_t)L * T, sizeof(double));
    double *betas = (double *)calloc((size_t)L * T, sizeof(double));
    double *ab = (double *)malloc((size_t)L * T * sizeof(double));
    double *absum = (double *)malloc((size_t)T * sizeof(double));
    double c, llForward, llBackward, tmp;
    int t, s, skip = 0;
    memset(grad, 0, (size_t)K * T * sizeof(double));

    A(0, 0) = 1.0;                                             /* :43 */
    llForward = log(P(seq[0], 0));                             /* :44 */
    for (t = 1; t < T && !skip; ++t) {                         /* :45-59 */
        for (s = 0; s < L; ++s) {
            if (s == 0) A(s, t) = A(s, t - 1) * P(s, t);
            else A(s, t) = (A(s, t - 1) + A(s - 1, t - 1)) * P(seq[s], t);
        }
        c = 0.0;
        for (s = 0; s < L; ++s) c += A(s, t);
        if (c == 0.0) { skip = 1; break; }
        for (s = 0; s < L; ++s) A(s, t) = A(s, t) / c;
        llForward += log(c);
    }
    if (!skip) {
        B(L - 1, T - 1) = 1.0;                                 /* :64 */
        llBackward = log(P(seq[L - 1], T - 1));
        for (t = T - 2; t >= 0 && !skip; --t) {                /* :66-82 */
            for (s = L - 1; s >= 0; --s) {
                if (s == L - 1) B(s, t) = B(s, t + 1) * P(seq[s], t);
                else B(s, t) = (B(s, t + 1) + B(s + 1, t + 1)) * P(seq[s], t);
            }
            c = 0.0;
            for (s = 0; s < L; ++s) c += B(s, t);
            if (c == 0.0) { skip = 1; break; }
            for (s = 0; s < L; ++s) B(s, t) = B(s, t) / c;
            llBackward += log(c);
        }
        (void)llBackward;
    }
    if (!skip) {
        for (t = 0; t < T; ++t)                                /* :85-87 */
            for (s = 0; s < L; ++s) AB(s, t) = A(s, t) * B(s, t);
        for (s = 0; s < L && !skip; ++s)                       /* :88-92 */
            for (t = 0; t < T; ++t) {
                G(seq[s], t) += AB(s, t);
                if (AB(s, t) != 0) {
                    if (P(seq[s], t) == 0.0) { skip = 1; break; }
                    AB(s, t) = AB(s, t) / P(seq[s], t);
                }
            }
    }
    if (!skip) {
        for (t = 0; t < T; ++t) {                              /* :94-97 */
            absum[t] = 0;
            for (s = 0; s < L; ++s) absum[t] += AB(s, t);
        }
        for (t = 0; t < T; ++t)                                /* :100-106 */
            for (s = 0; s < K; ++s) {
                tmp = P(s, t) * absum[t];
                if (tmp > 0) G(s, t) = P(s, t) - G(s, t) / tmp;
                else G(s, t) = P(s, t);
            }
    }
    *nll = -llForward;
    free(alphas); free(betas); free(ab); free(absum);
    return skip;
}

/*
 * The blank-forced loss and gradient in the log domain: float64 log-sum-exp recursions with no per-frame scaling, so
 * neither a state nor a product of alpha and beta leaves float64's range.  The reference's contract is kept, with "0"
 * meaning -inf, not underflow:
 *   alpha(0,0) = 1 with no emission, and the loss starts from log p[seq[0],0] (:43-44);
 *   state 0 takes row 0 in the alpha pass only (:49); beta(L-1,T-1) = 1 with no emission (:64);
 *   -nll = log p[seq[0],0] + log of the mass of ALL states at T-1 (the product of the frame normalisers);
 *   grad[k,t] = p - sum_{s: seq[s]=k} ab(s,t) / (p[k,t] * sum_s ab(s,t)/p[seq[s],t]) where p[k,t] * that sum > 0,
 *               else p (:100-106);
 *   skip, gradient all zeros: a normaliser of either pass is 0 (:108-110: all states -inf at some frame), or
 *               ab(s,t) != 0 where p[seq[s],t] == 0 (:88-92).  An utterance with no frame or no state also skips.
 * On skip *nll is the forward pass's (+inf when the forward mass is 0); the reference's partial llForward is not kept.
 */
int ctc_oracle_loss_blankforce_log(const double *params, int K, int T, const int *seq, int seqLen,
                                   double *grad, double *nll)
{
    int L = seqLen, t, s, k, skip = 0;
    double *la, *lb, *lp, *w, logZ;
    memset(grad, 0, (size_t)K * (T > 0 ? T : 0) * sizeof(double));
    if (T <= 0 || L <= 0) { *nll = 0.0; return 1; }
    la = (double *)malloc((size_t)L * T * sizeof(double));
    lb = (double *)malloc((size_t)L * T * sizeof(double));
    lp = (double *)malloc((size_t)K * T * sizeof(double));
    w = (double *)malloc((size_t)L * sizeof(double));
    for (t = 0; t < T; t++)
        for (k = 0; k < K; k++) lp[(size_t)k + (size_t)K * t] = log(P(k, t));
#define LP(k, t) lp[(size_t)(k) + (size_t)K * (size_t)(t)]
#define LA(s, t) la[(size_t)(s) + (size_t)L * (size_t)(t)]
#define LB(s, t) lb[(size_t)(s) + (size_t)L * (size_t)(t)]
    for (s = 0; s < L; s++) LA(s, 0) = (s == 0) ? 0.0 : -INFINITY;
    for (t = 1; t < T; t++)
        for (s = 0; s < L; s++)
            LA(s, t) = (s == 0) ? LA(0, t - 1) + LP(0, t) : lse2(LA(s, t - 1), LA(s - 1, t - 1)) + LP(seq[s], t);
    logZ = -INFINITY;
    for (s = 0; s < L; s++) logZ = lse2(logZ, LA(s, T - 1));
    *nll = -(LP(seq[0], 0) + logZ);
    if (logZ == -INFINITY) { skip = 1; goto done; }  /* the forward mass is 0 from some frame on */

    for (s = 0; s < L; s++) LB(s, T - 1) = (s == L - 1) ? 0.0 : -INFINITY;
    for (t = T - 2; t >= 0; t--) {
        double any = -INFINITY;
        for (s = L - 1; s >= 0; s--) {
            LB(s, t) = ((s == L - 1) ? LB(s, t + 1) : lse2(LB(s, t + 1), LB(s + 1, t + 1))) + LP(seq[s], t);
            any = any > LB(s, t) ? any : LB(s, t);
        }
        if (any == -INFINITY) { skip = 1; goto done; }
    }

    for (t = 0; t < T; t++) {
        double m = -INFINITY, q = 0.0;
        for (s = 0; s < L; s++) {
            double e = LA(s, t) + LB(s, t);
            w[s] = -INFINITY;
            if (e == -INFINITY) continue;
            if (P(seq[s], t) == 0.0) { skip = 1; goto done; }
            w[s] = e - LP(seq[s], t);
            m = w[s] > m ? w[s] : m;
        }
        if (m == -INFINITY) {                            /* absum == 0: the row stays p */
            for (k = 0; k < K; k++) G(k, t) = P(k, t);
            continue;
        }
        for (s = 0; s < L; s++) q += exp(w[s] - m);
        for (s = 0; s < L; s++) G(seq[s], t) += exp(w[s] - m) / q;
        for (k = 0; k < K; k++) G(k, t) = (P(k, t) > 0.0) ? P(k, t) - G(k, t) : P(k, t);
    }
done:
    if (skip) memset(grad, 0, (size_t)K * T * sizeof(double));
#undef LP
#undef LA
#undef LB
    free(la); free(lb); free(lp); free(w);
    return skip;
}

/* ctc_fast_blankforce.pyx:115-142: argmax per frame, drop blanks and repeats (no label filter, no
 * alignment output).  Returns the hypothesis length. */
int ctc_oracle_best_path_blankforce(const double *probs, int K, int T, int blank, int *hyp)
{
    int n = 0, prev = -1, t;
    for (t = 0; t < T; ++t) {
        int b = argmax_frame(probs, K, t);
        if (b != blank && !(t != 0 && b == prev)) hyp[n++] = b;
        prev = b;
    }
    return n;
}
