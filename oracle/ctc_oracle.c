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

int ctc_oracle_loss(const double *params, int K, int T, const int *seq, int seqLen,
                    int blank, double *grad, double *nll)
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
    (void)llBackward;

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
    free(alphas); free(betas); free(ab); free(absum);
    return skip;
}

/* ctc_fast.pyx:154-187 -- per-frame argmax, collapse repeats, drop blank and labels 1,2,8.
 * hyp/align must hold T ints; returns the hypothesis length. */
int ctc_oracle_best_path(const double *probs, int K, int T, int blank, int *hyp, int *align)
{
    int n = 0, prev = -1, t, k;
    for (t = 0; t < T; t++) {
        int b = 0;
        double m = probs[(size_t)K * t];
        for (k = 1; k < K; k++)
            if (probs[(size_t)k + (size_t)K * t] > m) { m = probs[(size_t)k + (size_t)K * t]; b = k; }
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

/* ctc_fast_blankforce.pyx:115-142: argmax per frame, drop blanks and repeats (no label filter, no
 * alignment output).  Returns the hypothesis length. */
int ctc_oracle_best_path_blankforce(const double *probs, int K, int T, int blank, int *hyp)
{
    int n = 0, prev = -1, t, k;
    for (t = 0; t < T; ++t) {
        int b = 0;
        for (k = 1; k < K; ++k)
            if (probs[(size_t)k + (size_t)K * t] > probs[(size_t)b + (size_t)K * t]) b = k;
        if (b != blank && !(t != 0 && b == prev)) hyp[n++] = b;
        prev = b;
    }
    return n;
}
