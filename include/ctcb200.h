/*
 * ctcb200.h -- C ABI of libctcb200.so, the H100 (sm_90a) compute backend for the
 * stanford-ctc training hot path (BRNN forward/backward + CTC alpha/beta + Nesterov SGD).
 *
 * Every entry point takes plain pointers and sizes (no torch types).  Unless a parameter is
 * documented as a HOST pointer it is a DEVICE pointer; all work is enqueued asynchronously on
 * the caller-supplied cudaStream_t (passed as void*).  Return value: 0 on success, a negative
 * CTCB_E* code otherwise, with a message retrievable from ctcb_last_error().  Numerical
 * infeasibility of one utterance (the reference's `skip=True`) is NOT an error: it is reported
 * per utterance in `skip_out`, as ctc_fast/ctc-loss/ctc_fast.pyx:147-149 does.
 *
 * The reference interface each entry point replaces is cited as (file:line) relative to
 * the original stanford-ctc checkout.
 */
#ifndef CTCB200_H
#define CTCB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTCB_OK 0
#define CTCB_EINVAL (-1)   /* bad argument / unsupported shape */
#define CTCB_ECUDA (-2)    /* CUDA runtime error (see ctcb_last_error) */
#define CTCB_ENOMEM (-3)   /* caller workspace too small */

/* Longest label sequence per utterance the CTC kernel accepts (16 state pairs per lane, ctc.cu). */
#define CTCB_CTC_MAX_LABELS 511

/* ---- library ------------------------------------------------------------------------------ */
int ctcb_version(void);
const char *ctcb_last_error(void);
/* Number of kernels this library has launched since it was loaded (bench.py: gpu_launches). */
uint64_t ctcb_launch_count(void);
/* Per-phase device timing with CUDA events on the launching stream (bench.py roofline). When enabled,
 * every phase of ctcb_brnn_cost_and_grad and the optimiser entry points is bracketed by events;
 * ctcb_profile_report synchronises the device and writes a JSON object
 * {"phase": {"count": n, "total_ms": t}, ...} into buf, then clears the records. */
void ctcb_profile_enable(int on);
int ctcb_profile_report(char *buf, size_t cap);

/* ---- CTC loss + gradient (replaces ctc_fast.ctc_loss, ctc_fast/ctc-loss/ctc_fast.pyx:13-152;
 *      call site ctc_fast/nnets/brnnet.py:175, with the softmax of brnnet.py:161-168 fused) ----
 * acts      : activations of B utterances; element (u, t, k) at acts[u*utt_stride + t*frame_stride + k]
 *             (strides in elements).  is_prob=0: pre-softmax logits, the softmax is fused;
 *             is_prob=1: probabilities (the contract of ctc_fast.ctc_loss's `params`).
 * labels    : concatenated int32 label sequences; utterance u owns labels[label_off[u] .. label_off[u+1])
 * T_per_utt : int32[B] frame counts (<= Tmax).  Frames t >= T_per_utt[u] get zero gradient.
 * grad_out  : same indexing as acts; d(nll)/d(logit) = softmax - posterior occupancy
 *             (ctc_fast.pyx:139-145).  Zero for skipped utterances.
 * nll_out   : float32[B]  -log p(labels | acts)     (ctc_fast.pyx:152)
 * skip_out  : int32[B]    1 where a frame normaliser was 0 (ctc_fast.pyx:147-149), and 1 where the scaled trellis
 *             lost mass to float64 underflow (forward and backward log-likelihoods more than 1e-4 nats apart: long
 *             utterances with unaligned outputs, where the reference returns a wrong loss and gradient), and,
 *             checked on the device before any row is read, where utterance u is malformed: a label count
 *             label_off[u+1] - label_off[u] below 0 or above max_labels, or a label outside [0, K).  A malformed
 *             utterance is skipped exactly as one with T_per_utt = 0: the same nll, a zero gradient on all Tmax rows.
 * workspace: ctcb_ctc_workspace_bytes(B, Tmax, max_labels) bytes of device scratch.  That size never decreases with B,
 *             Tmax or max_labels, so a buffer sized for the largest call serves every smaller one: one fp64 trellis
 *             plane of Tmax x 64P doubles (P = pairs per lane, 1..16 by max_labels) per utterance, two per utterance
 *             for the first 256 (the frame-parallel kernel spills alpha and beta), i.e. max(B, 2 min(B, 256)) planes.
 */
size_t ctcb_ctc_workspace_bytes(int B, int Tmax, int max_labels);
int ctcb_ctc_loss_grad_f32(const float *acts, int is_prob, int64_t utt_stride, int64_t frame_stride,
                           const int32_t *labels, const int32_t *label_off, const int32_t *T_per_utt,
                           int B, int Tmax, int K, int max_labels, int blank,
                           float *grad_out, float *nll_out, int32_t *skip_out,
                           void *workspace, size_t ws_bytes, void *stream);

/* ---- best-path decode (replaces ctc_fast.decode_best_path, ctc_fast.pyx:154-187) -----------
 * hyp_out/align_out: int32[B*Tmax] (row u holds hyp_len_out[u] valid entries).
 * The label of a frame is np.argmax's: the first NaN if there is one, else the first maximum (0 for a row of -inf).
 * drop_swbd_noise!=0 reproduces the reference's removal of labels 1, 2 and 8 (ctc_fast.pyx:176-179). */
int ctcb_ctc_best_path_f32(const float *acts, int64_t utt_stride, int64_t frame_stride,
                           const int32_t *T_per_utt, int B, int Tmax, int K, int blank,
                           int drop_swbd_noise, int32_t *hyp_out, int32_t *align_out,
                           int32_t *hyp_len_out, void *stream);

/* ---- blank-forced CTC (replaces ctc_fast_blankforce.ctc_loss, ctc-loss/ctc_fast_blankforce.pyx:13-113) ----
 * Same buffers as ctcb_ctc_loss_grad_f32, but `seq` already contains the blanks (:24-26): utterance u has
 * seq_off[u+1]-seq_off[u] trellis states (at most 1024), moves s->s and s->s+1 only, one start and one end
 * state, no window; state 0 is propagated with row 0 of the probabilities (:49).  grad_out must not alias
 * acts.  workspace: ctcb_ctc_blankforce_workspace_bytes(B, Tmax, max_states) bytes (the log-alpha trellis).
 * The recursions run in the log domain, so unlike the reference the result stays right on long utterances whose
 * normalised trellis products underflow float64.  skip_out[u] = 1 with a zero gradient where the reference skips (a
 * zero frame normaliser, or alpha*beta != 0 where the state's probability is 0), and, checked on the device before
 * any state is read, where utterance u has T_per_utt <= 0, no state, more states than max_states, or a label outside
 * [0, K).  The launch refuses (CTCB_EINVAL) max_states outside 1..1024 and 20*max_states + 256 + 8*K > 200 KiB of
 * shared memory: K <= 25565 at max_states = 1, K <= 23008 at 1024.
 * The best path of that module (:115-142) is ctcb_ctc_best_path_f32 with drop_swbd_noise=0; its align
 * output is simply not used. */
size_t ctcb_ctc_blankforce_workspace_bytes(int B, int Tmax, int max_states);
int ctcb_ctc_blankforce_loss_grad_f32(const float *acts, int is_prob, int64_t utt_stride, int64_t frame_stride,
                                      const int32_t *seq, const int32_t *seq_off, const int32_t *T_per_utt,
                                      int B, int Tmax, int K, int max_states,
                                      float *grad_out, float *nll_out, int32_t *skip_out,
                                      void *workspace, size_t ws_bytes, void *stream);

/* ---- dense fp32 contraction (replaces cudamat cm.dot call sites brnnet.py:140,196,204,227-230) ----
 * Row-major C[M x N] = alpha * op(A) * op(B) + beta * C, op(X) = X or X^T per transA/transB.
 * A is M x K (or K x M if transA), leading dimensions in elements.
 * bias (may be NULL): added per output column n.  relu!=0: C = max(C, 0) after bias.
 * mask_src (may be NULL, ldc-strided like C): C *= (mask_src > 0).
 * workspace is used for split-K partial sums (ctcb_gemm_workspace_bytes).  M is at most 8,388,480 (65,535 tiles of
 * 128 rows); a larger M returns CTCB_EINVAL.  K is not limited. */
size_t ctcb_gemm_workspace_bytes(int M, int N, int K);
int ctcb_gemm_f32(int transA, int transB, int M, int N, int K, float alpha,
                  const float *A, int64_t lda, const float *B, int64_t ldb, float beta,
                  float *C, int64_t ldc, const float *bias, int relu, const float *mask_src,
                  void *workspace, size_t ws_bytes, void *stream);
/* Two contractions of one shape, pitches, alpha and beta (no bias, ReLU or mask): C0 = op(A0) op(B0), C1 = op(A1) op(B1).
 * On the tensor cores both share one launch and one split-K reduce when every operand can be read in place; each
 * result is then the same as that of the single call at the same split.  Otherwise two ctcb_gemm_f32 calls. */
size_t ctcb_gemm_pair_workspace_bytes(int M, int N, int K);
int ctcb_gemm_pair_f32(int transA, int transB, int M, int N, int K, float alpha,
                       const float *A0, const float *A1, int64_t lda, const float *B0, const float *B1, int64_t ldb,
                       float beta, float *C0, float *C1, int64_t ldc, void *workspace, size_t ws_bytes, void *stream);
/* The plan ctcb_gemm_f32 (problems = 1) or ctcb_gemm_pair_f32 (problems = 2) runs for these arguments under the
 * knobs in effect (INTEGRATION.md section 4), assuming a large enough workspace.  A and B are only
 * inspected for their alignment.  out (HOST, 8 int32):
 *   {kernel: 0 FFMA / 1 tensor core, BN (output tile width), ring stages, K splits, CTAs per launch,
 *    A path, B path: 0 read in place K-major / 1 read in place MN-major, transposed in shared memory / 2 copied into
 *    the workspace first,  problems per launch (2: the pair shares one launch)}.  The FFMA kernel reports
 *   {0, 128, 0, K splits, CTAs per launch, vec, 0, 1}: vec (in the A path slot) = 1 when both operands are read with
 *   16-byte loads (both pitches multiples of 4 floats, both bases 16-byte aligned); each split accumulates
 *   ceil(K / splits) rounded up to a multiple of 16.  M <= 0 or N <= 0 reports {0, .., 0, 1}. */
int ctcb_debug_gemm_plan(int transA, int transB, int M, int N, int K, const float *A, int64_t lda,
                         const float *B, int64_t ldb, int problems, int32_t *out);
/* The same three in TF32 mode (ctcb_brnn_config.tf32, below): same arguments and workspace; a shape that goes to the
 * FFMA kernel runs it, with ctcb_gemm_f32's bits, and the plan entry reports it.  The TF32 plans keep the default's
 * BN, K splits and operand paths; their ring stages are their own. */
int ctcb_gemm_tf32(int transA, int transB, int M, int N, int K, float alpha,
                   const float *A, int64_t lda, const float *B, int64_t ldb, float beta,
                   float *C, int64_t ldc, const float *bias, int relu, const float *mask_src,
                   void *workspace, size_t ws_bytes, void *stream);
int ctcb_gemm_pair_tf32(int transA, int transB, int M, int N, int K, float alpha,
                        const float *A0, const float *A1, int64_t lda, const float *B0, const float *B1, int64_t ldb,
                        float beta, float *C0, float *C1, int64_t ldc, void *workspace, size_t ws_bytes, void *stream);
int ctcb_debug_gemm_plan_tf32(int transA, int transB, int M, int N, int K, const float *A, int64_t lda,
                              const float *B, int64_t ldb, int problems, int32_t *out);

/* Debug hook: set one planner knob of INTEGRATION.md section 4 in this process, e.g. ("CTCB_CTC", "ckpt") or
 * ("CTCB_SWEEP_TC_CS", "2").  value uses the environment's syntax; value == NULL restores what the environment said at
 * the library's first use, or the default.  An unknown name or a value outside the documented set returns CTCB_EINVAL
 * and changes nothing.  Do not call it while other threads make library calls.  A change takes effect at the next
 * planning call.  Workspace sizes, and the forward layout a net handle caches, reflect the knobs in effect when they
 * were computed (ctcb_gemm_workspace_bytes depends on CTCB_GEMM): set knobs before sizing workspaces or creating nets. */
int ctcb_debug_set_knob(const char *name, const char *value);

/* Diagnostic / measurement: force the CTC kernel organisation used by ctcb_ctc_loss_grad_f32 (and the BRNN step).
 * 0 = automatic (by batch size), 1 = one warp per utterance with the trellis spilled to the workspace, 2 = two warps per
 * utterance meeting in the middle, 3 = recurrences on two warps + frame-parallel gradient (at most 256 utterances),
 * 4 = one warp per utterance with on-chip checkpoints (at most 127 labels).  Same as ctcb_debug_set_knob("CTCB_CTC",
 * "auto" | "warp" | "pair" | "par" | "ckpt").  A forced organisation that cannot run these arguments
 * (par beyond 256 utterances, par / pair / ckpt with K too large for their tiles, ckpt beyond 127 labels) makes
 * ctcb_ctc_loss_grad_f32 return CTCB_EINVAL; it never runs another one.  Probability input (is_prob = 1) gives the same
 * bits whichever organisation runs.  Logits give the same bits within a tile height -- 16 frames: par, pair, and warp
 * below 16 x SMs utterances or beyond 63 labels; 8 frames: ckpt, and warp otherwise -- but the fused softmax sums a
 * row's normaliser in another order in the two, so across them the gradient and the loss differ in the last bits. */
int ctcb_debug_set_ctc_kernel(int shape);
/* The plan ctcb_ctc_loss_grad_f32 runs for these arguments under the organisation in effect (CTCB_CTC /
 * ctcb_debug_set_ctc_kernel) and the device's SM count.  acts and grad_out are inspected only for their alignment.
 * out (HOST, 8 int32): {kernel: 0 par / 1 pair / 2 ckpt / 3 warp, P (pairs per lane), frames per time tile,
 * activation tiles per warp, warps per CTA (par: the warps of its gradient phase), vec2 (8-byte tile copies and
 * stores), shared row pitch in floats, dynamic shared memory per CTA in KiB rounded up}.  Returns the error the call
 * itself would return for these sizes (e.g. K too large for the tile), assuming valid pointers, blank and workspace. */
int ctcb_debug_ctc_plan(int B, int Tmax, int K, int max_labels, const float *acts, const float *grad_out,
                        int64_t utt_stride, int64_t frame_stride, int32_t *out);

/* Diagnostic (CTCB_GEMM_TRACE=1): SM clock stamps of CTA (0,0,0) of the last tensor-core GEMM, HOST buffer of 64 x 8
 * uint64 = per k-block {TMA issued, tile landed, low halves written, MMA thread saw it, MMAs issued, -, -, -}. */
int ctcb_debug_gemm_trace(unsigned long long *host_out);

/* ---- BRNN (replaces nnets.brnnet.NNet, ctc_fast/nnets/brnnet.py:10-277) --------------------- */
typedef struct ctcb_brnn_config {
    int32_t inputDim;      /* brnnet.py:10 */
    int32_t outputDim;
    int32_t layerSize;
    int32_t numLayers;
    int32_t temporalLayer; /* <=0: none.  1..numLayers (numLayers itself is an extension, see DESIGN.md) */
    int32_t maxT;          /* frames per utterance the buffers are sized for (reference: maxBatch) */
    int32_t maxB;          /* utterances per step; maxT * maxB is at most 8,388,480 (the rows of a ctcb_gemm_f32), else
                            * the config is invalid */
    int32_t maxLabels;     /* longest label sequence */
    float reg;             /* L2 coefficient (brnnet.py:11,177-183,197-198,244-247) */
    float maxAct;          /* clip of the temporal layer, 20.0 (brnnet.py:32) */
    int32_t unidirectional; /* 0: nnets/brnnet.py (Wtf and Wtb, output For+Back).  1: nnets/rnnet.py:91-191 -- one
                             * recurrent matrix, forward in time only, stack = [...layers, [Wt, dummy]] (rnnet.py:57-65).
                             * temporalLayer <= 0 with either value is the plain DNN of nnets/nnet.py:57-113. */
    int32_t numTemporal;   /* k: layers temporalLayer .. temporalLayer+k-1 are all temporal, each with its own recurrent
                            * matrices and sweeps (output For_j + Back_j, uni-directional For_j).  0 and 1 both mean
                            * one temporal layer, so an initialiser without this member keeps its meaning.  k > 1 needs
                            * 1 <= temporalLayer and temporalLayer + k - 1 <= numLayers, else the config is invalid. */
    int32_t cell;          /* recurrence of every temporal layer: 0 the reference's clipped ReLU (so an initialiser without
                            * this member keeps its meaning), 1 LSTM (below); any other value makes the config invalid. */
    int32_t layerNorm;     /* 0: off (so an initialiser without this member keeps its meaning); 1: layer normalisation of
                            * the ReLU hidden layers (below); any other value makes the config invalid. */
    int32_t subsample;     /* k: 0 and 1 off (so an initialiser without this member keeps its meaning); k >= 2 runs affine
                            * map subsampleLayer and everything above it at 1/k of the input frame rate (below); a
                            * negative value makes the config invalid. */
    int32_t subsampleLayer; /* L: ignored for k <= 1; with k >= 2 it needs 1 <= L <= numLayers + 1, else the config is
                             * invalid. */
    int32_t peephole;      /* 0: off (so an initialiser without this member keeps its meaning); 1: peephole connections of
                            * the LSTM cell (below), which needs cell = 1; any other value, or 1 with cell = 0, makes the
                            * config invalid.  Without a temporal layer it lays out and launches nothing. */
    int32_t maskFeatDim;   /* nu: 0 off (so an initialiser without this member keeps its meaning); nu > 0 lays the input
                            * rows out as c = inputDim / nu frame slots of nu filter-bank bins for the SpecAugment masks
                            * of ctcb_brnn_set_input_masks (below) and reserves their masked copy in the training
                            * workspace.  Invalid: nu < 0, nu not dividing inputDim, an even c, or a layout whose bit sets
                            * exceed the mask pass's 48 KB of shared memory (about inputDim + 64 > 393,000 bits). */
    int32_t weightNoise;   /* 0: off (so an initialiser without this member keeps its meaning); 1: reserves the noisy copy
                            * of the parameters for the Gaussian weight noise of ctcb_brnn_set_weight_noise (below) in
                            * the training workspace; any other value makes the config invalid. */
    int32_t zoneout;       /* 0: off (so an initialiser without this member keeps its meaning); 1: zoneout of the LSTM
                            * cell's state (below) with the probabilities of ctcb_brnn_set_zoneout, which needs cell = 1;
                            * any other value, or 1 with cell = 0, makes the config invalid. */
    int32_t interLayer;    /* m: 0 off (so an initialiser without this member keeps its meaning); 1 <= m <= numLayers - 1
                            * adds the intermediate CTC loss of hidden layer m to training calls (below); any other value
                            * makes the config invalid. */
    float interWeight;     /* lambda of the intermediate CTC loss: ignored with interLayer = 0; with interLayer > 0 a
                            * value that is not finite and > 0 makes the config invalid. */
    int32_t selfCondition; /* 0: off (so an initialiser without this member keeps its meaning); 1: self-conditioned CTC
                            * (below), which needs interLayer >= 1; any other value, or 1 with interLayer = 0, makes the
                            * config invalid. */
    int32_t tf32;          /* 0: off (so an initialiser without this member keeps its meaning); 1: every tensor-core
                            * contraction and sweep of the net's training and forward-only calls runs in TF32 mode
                            * (below); any other value makes the config invalid. */
} ctcb_brnn_config;

/* TF32 mode (tf32 = 1, ctcb_gemm_tf32, ctcb_brnn_sweep_tf32; not in the reference).  By default every product on the
 * tensor cores is fp32-faithful: each operand is split into two TF32 parts and a product costs three MMAs (3xTF32).
 * In TF32 mode every product that runs on the tensor cores reads each operand rounded to the nearest TF32 value, ties
 * away from zero (cvt.rna.tf32.f32: the low 13 mantissa bits become zero), and is ONE .tf32 MMA accumulated in fp32, as
 * PyTorch's allow_tf32 does.  The K splits (no accumulator chain longer than K = 2048) and the deterministic split-K
 * reduce are those of the default, and so are the workspace sizes and offsets: ctcb_gemm_workspace_bytes,
 * ctcb_brnn_sweep_workspace_bytes, ctcb_brnn_workspace_bytes and ctcb_brnn_forward_workspace_bytes do not depend on
 * the mode.  The exact FFMA kernels keep their bits in either mode: the small contractions (ctcb_debug_gemm_plan
 * kernel 0), the cluster and generic ReLU sweeps (H <= 512), the LSTM sweeps, the CTC, layer normalisation and the
 * optimisers.  No parameter changes, so checkpoints are the same in both modes. */

/* Intermediate CTC loss (interLayer = m >= 1; not in the reference; Lee & Watanabe, "Intermediate Loss Regularization
 * for CTC-based Speech Recognition", ICASSP 2021, after the hierarchical CTC of Fernandez et al. 2007 and Sanabria &
 * Metze, SLT 2018).  N = numLayers, K = outputDim, lambda = interWeight.  X_m is hidden layer m's output as map m + 1
 * sees it (dropped, normalised, For + Back at a bi-directional temporal layer, h_f + h_b at an LSTM layer), on T_m
 * frames: T_u, or T'_u = ceil(T_u / k) when m >= subsampleLayer.  The head is the net's own output map, as in ESPnet's
 * InterCTC; it adds no parameter, so the flat vector, checkpoints and forward-only calls are those of the net without it.
 *   Forward (training calls only): A = X_m W_{N+1}^T + b_{N+1}, [T_m][B][K]; nll_aux[u] is the CTC loss of softmax(A)
 *   against utterance u's labels over its T_m frames, with the blank, maxLabels and skip rules of the main CTC.
 *   Objective: cost = nll_main + lambda nll_aux per utterance.  Lee & Watanabe's (1 - w) L + w L_inter is this objective
 *   with lambda = w / (1 - w) and the step size scaled by (1 - w); this form leaves the gradient of the top of the net
 *   as it is without the loss.
 *   Backward: D_aux = lambda d(nll_aux)/dA (the CTC gradient scaled in place, once, so that the two contractions and the
 *   column sums below read the same values); dW_{N+1} += D_aux^T X_m and db_{N+1} += the column sums of D_aux; the
 *   incoming delta of layer m gains D_aux W_{N+1}, under the ReLU mask and dropout's alpha of the delta from map m + 1,
 *   added before layer normalisation's backward or the BPTT sweep reads it (behind the unstacking when map m + 1 reads
 *   stacked frames: the term is at layer m's own rate).
 *   Each CTC skips on its own: an utterance the intermediate CTC skips gets no gradient from it and adds nothing to its
 *   sums.  cost_out, skip_out and the first four floats of stats_out keep their meaning (the main CTC's).
 * Forward-only calls (grads == NULL) never run the head, unless selfCondition = 1 (below): probs_out and the forward
 * workspace are those of the net without it.  Invalid configs: m outside 0..N-1, lambda not finite and > 0 with m > 0, and m > 0 with subsample >= 2
 * at subsampleLayer = N + 1 (W_{N+1} then reads k H columns and cannot take X_m).
 *
 * Self-conditioned CTC (selfCondition = 1 with interLayer = m; not in the reference; Nozaki & Komatsu, "Relaxing the
 * Conditional Independence Assumption of CTC-based ASR by Conditioning on Intermediate Predictions", Interspeech 2021;
 * ESPnet's interctc_use_conditioning).  H = layerSize.  The intermediate posteriors are projected back to the layer's
 * width and added to its output, so the layers above condition on a first guess at the labels.  Parameters W_c (H x K)
 * and b_c (H), behind every other tensor of the flat vector (below).
 *   Forward (training and forward-only calls): A = X_m W_{N+1}^T + b_{N+1} (as above); P = softmax(A) per row (float32,
 *   the row-softmax kernel); X'_m = X_m + P W_c^T + b_c.  Map m + 1 reads X'_m in place of X_m, and so does the frame
 *   stacking when m + 1 = subsampleLayer.  The intermediate CTC still scores A.  X_m keeps every other role: the ReLU
 *   and dropout mask of layer m's delta and the head's input.  A training call writes X'_m into a buffer of its own,
 *   a forward-only call over X_m in place, with the same launches and plans, so probs_out stays bit-identical.
 *   Backward: D'_m = dL/dX'_m is the delta contraction of map m + 1 (after any unstacking), without the mask and with
 *   alpha = 1.  dP = D'_m W_c; dA = P (dP - sum_k P_k dP_k) + D_aux (ctcb_softmax_rows_backward_f32); dW_c = D'_m^T P,
 *   db_c = the column sums of D'_m; dW_{N+1} += dA^T X_m and db_{N+1} += the column sums of dA (in place of the D_aux
 *   term above); the delta of layer m is alpha [X_m > 0] (D'_m + dA W_{N+1}), the mask and alpha at a ReLU layer only,
 *   and layer normalisation's backward or the BPTT sweep read it as they read the delta without conditioning.
 *   W_c and b_c start at 0 (a new net is the InterCTC net), are not L2-regularised and get no weight noise.  The
 *   objective is still nll_main + lambda nll_aux. */

/* Frame subsampling (subsample = k >= 2; not in the reference; cf. Deep Speech 2's striding and the frame stacking of
 * pyramidal and low-frame-rate CTC models).  Affine map L = subsampleLayer reads k consecutive frames of layer L - 1
 * concatenated: the input features when L = 1, else that layer's activations as the next map sees them without
 * subsampling (dropped, normalised, For + Back, ...).  Utterance u has T'_u = ceil(T_u / k) frames from map L upward,
 * and a call with Tmax has Tmax' = ceil(Tmax / k):
 *   S[t'] = [x_{k t'}, x_{k t' + 1}, ..., x_{k t' + k - 1}]   (frame-major: unit j of sub-frame m is column m n + j)
 *   with x_t = 0 for t >= T_u (not the padded row's content), so W_L is rows(L) x k n.
 * Maps L .. numLayers + 1, their temporal layers (both cells, both directions: the sweeps start and end at T'_u, the
 * recurrent weight gradients use the rows shifted by B of the reduced-rate buffers), the softmax and the CTC run on
 * T'_u frames.  probs_out of a forward-only call is [Tmax'][B][outputDim].  The CTC skips an utterance it cannot align
 * in T'_u frames as it does in T_u.  Dropout keeps its definition with t the frame at the layer's own rate (t' for
 * layers >= L); layer normalisation is per row and unchanged.  The flat vector keeps its tensor count and order; only
 * W_L widens.  Backward: dS = (W_L^T delta_L) * (S > 0) where layer L - 1 is a ReLU hidden layer (with dropout's
 * alpha), unmasked at a temporal layer; then D[t][u][j] = dS[t / k][u][(t % k) n + j] for t < T_u, 0 beyond;
 * dW_L = delta_L^T S. */

/* Layer normalisation (layerNorm = 1; not in the reference; Ba, Kiros & Hinton 2016).  Hidden layer i is normalised
 * when 1 <= i <= numLayers and i is not temporal -- exactly the layers dropout drops.  Per frame row, H = layerSize:
 *   z = W_i x + b_i;  mu = mean_j z_j;  var = mean_j (z_j - mu)^2 (biased);  rstd = 1 / sqrt(var + 1e-5)
 *   xh = (z - mu) rstd;  X_i = relu(gamma_i xh + beta_i)      (then inverted dropout, unchanged, when p > 0)
 * i.e. torch.nn.functional.layer_norm with eps = 1e-5, then ReLU.  The input, the temporal layers and the logits are
 * never normalised; padded frames are normalised like any row (their delta is 0, so they add nothing to a gradient).
 * Backward, g = dL/d(gamma xh + beta) (the masked delta contraction, with dropout's alpha), gh = g gamma:
 *   dz = rstd (gh - mean_j gh - xh mean_j(gh xh));  dgamma = sum over rows of g xh;  dbeta = sum over rows of g.
 * Each normalised layer adds [gamma_i, beta_i], each H x 1, behind every other tensor of the flat vector, in layer
 * order; gamma and beta are not L2-regularised.  Statistics are fp32, the mean first and then the squared deviations
 * from it, in an order that depends only on H.  layerSize above CTCB_LAYERNORM_MAX_H makes such a config invalid. */
#define CTCB_LAYERNORM_MAX_H 8192

/* The LSTM cell (cell = 1; not in the reference).  Temporal layer i with input width n, H = layerSize, ndir = 2
 * (bi-directional) or 1, G = ndir * 4H:
 *   affine map [W_i, b_i] is G x n and G x 1; rows 0..4H-1 belong to the forward-in-time direction, 4H..8H-1 to the
 *   backward one, each block in gate order i, f, g, o (torch.nn.LSTM's).  pre = W_i x + b_i.
 *   each recurrent matrix is U (4H x H), still followed by its 1-float dummy; tensor count and order are unchanged.
 *   per direction (the backward one mirrored in time), float32 with accurate expf / tanhf:
 *     z_t = pre_t + U h_{t-1};  i, f, o = sigmoid(z_i, z_f, z_o);  g = tanh(z_g);  c_t = f c_{t-1} + i g;  h_t = o tanh(c_t)
 *     h and c are 0 before the first frame and at every frame t >= T_u (the backward direction starts at T_u - 1);
 *     there is no clip and maxAct is ignored.
 *   layer output h_f + h_b (uni-directional: h_f), H wide.
 *   BPTT: dh_t = delta_t + U^T dz_{t+1};  dc_t = dh_t o (1 - tanh^2 c_t) + dc_{t+1} f_{t+1};
 *     dz = [dc g i(1-i), dc c_{t-1} f(1-f), dc i (1-g^2), dh tanh(c_t) o(1-o)];  dU = sum_t dz_t h_{t-1}^T,
 *     dW_i = sum_t dz_t x_t^T, db_i = sum_t dz_t, delta_{i-1} = W_i^T dz; L2 adds reg W to W_i and U as to every matrix.
 * ctcb_brnn_create refuses (CTCB_EINVAL, the message names the width) a layerSize whose sweep the device cannot hold
 * co-resident: ndir * ceil(H / 8) CTAs of 256 threads, at most two per SM (bi-directional H = 2048 on an H100). */

/* Peephole connections (peephole = 1 with cell = 1; Graves, Mohamed & Hinton 2013, eqs. 3-7; the cell of EESEN and of
 * Kaldi's nnet1 LSTM).  Per direction of every LSTM layer three H-vectors p_i, p_f, p_o; only the sigmoid gates change:
 *     i = sigmoid(z_i + p_i c_{t-1});  f = sigmoid(z_f + p_f c_{t-1});  g = tanh(z_g);  c_t = f c_{t-1} + i g;
 *     o = sigmoid(z_o + p_o c_t);  h_t = o tanh(c_t)
 *   (the backward-in-time direction mirrored: c_{t+1} in place of c_{t-1}).  c is 0 before the first frame and at every
 *   frame t >= T_u, as without peepholes.  The gates buffer holds o after its peephole.
 *   BPTT ("next" = t + 1 in the direction's order):
 *     dz_o = dh tanh(c_t) o(1-o);  dc_t = dh o (1 - tanh^2 c_t) + p_o dz_o + f_{t+1} dc_{t+1} + p_i dz_i,{t+1} + p_f dz_f,{t+1}
 *     dz_i, dz_f, dz_g as without peepholes, from this dc_t;
 *     dp_i = sum_{t,u} dz_i,t c_{t-1};  dp_f = sum dz_f,t c_{t-1};  dp_o = sum dz_o,t c_t   (padded frames add nothing).
 * Each LSTM layer adds one entry per direction, [P_d (3 x H, rows i, f, o), dummy (1 x 1)], in the recurrent entries'
 * order (temporal layers ascending, forward before backward), behind every other tensor of the flat vector (the
 * [gamma, beta] pairs included), so no other offset and not the early all-reduce range moves; the peephole gradients
 * travel with the exchange at the end of the step.  P is not L2-regularised; the dummies get a zero gradient. */

/* Zoneout (zoneout = 1 with cell = 1; not in the reference; Krueger et al., ICLR 2017).  For each LSTM temporal layer i
 * (its hidden-layer index, 1..numLayers) and direction d (0 forward in time, 1 backward), time in the direction's own
 * order (the backward direction mirrored, as above), frames at the layer's own rate, and the two probabilities z_c, z_h
 * in [0, 1) of ctcb_brnn_set_zoneout:
 *     c~_t = f_t c_{t-1} + i_t g_t;   c_t = lambda_c,t c_{t-1} + (1 - lambda_c,t) c~_t
 *     h~_t = o_t tanh(c_t);           h_t = lambda_h,t h_{t-1} + (1 - lambda_h,t) h~_t
 *   c and h are 0 before the first frame and at every frame t >= T_u, as without zoneout; with peepholes i and f see
 *   the zoned c_{t-1} and o the zoned c_t.  The layer's output is h_f + h_b (uni-directional h_f) of the zoned h, and
 *   the c buffers hold the zoned c.
 * Training calls (grads != NULL) draw lambda in {0, 1} for unit j of frame t of minibatch utterance g (as
 * ctcb_brnn_set_dropout_utts places it; t the frame index 0..T-1 at the layer's rate, in either direction) at step s:
 *     (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32, g mod 2^32, t, (i << 24) | (d << 23) | j),
 *                                      key = (seed mod 2^32, seed >> 32))
 *     lambda_c = 1 iff r0 < floor(z_c 2^32),  lambda_h = 1 iff r1 < floor(z_h 2^32)     (the products in float64)
 *   and lambda = 1 is a select: the kept value has exactly the bytes of c_{t-1} or h_{t-1}.  The counter never meets
 *   the other draws of a seed: dropout's fourth word carries a non-temporal layer's index in its top 8 bits, this
 *   rule's a temporal one's; SpecAugment's fourth word is < 2^24 and this rule's >= 2^24 (i >= 1); weight noise's
 *   fourth word is 0.
 * Forward-only calls (grads == NULL) use the expectation, lambda_c = z_c and lambda_h = z_h in float32:
 *   c_t = fmaf(z_c, c_{t-1}, (1 - z_c) c~_t), h_t likewise.  So with a probability > 0 a forward-only call's probs_out
 *   is not a training call's (ctcb_brnn_forward_workspace_bytes); at z_c = z_h = 0 nothing changes.
 * BPTT (training calls; "next" = t + 1 in the direction's order):
 *     dh_t  = delta_t + U^T dz_next + lambda_h,next dh_next;   dh~_t = (1 - lambda_h,t) dh_t
 *     dz_o  = dh~_t tanh(c_t) o(1-o)
 *     dc_t  = dh~_t o (1 - tanh^2 c_t) [+ p_o dz_o] + (lambda_c,next + (1 - lambda_c,next) f_next) dc_next
 *             [+ p_i dz_i,next + p_f dz_f,next];   dc~_t = (1 - lambda_c,t) dc_t
 *     dz_i = dc~_t g i(1-i);  dz_f = dc~_t c_{t-1} f(1-f);  dz_g = dc~_t i(1-g^2)
 *   dU, dW, db, delta_{i-1} and dP are unchanged and read the zoned h and c.  At lambda = 0 every formula is the cell
 *   above.  No tensor is added and the flat vector does not change. */

typedef struct ctcb_brnn ctcb_brnn; /* opaque; owns no device memory */

/* Flat parameter vector layout: the reference's `stack` order (brnnet.py:38-41,66-72):
 * [W1,b1] ... [W_{N+1},b_{N+1}] [Wtf,dummy] [Wtb,dummy]; W row-major (out x in), dummy = 1 float.
 * unidirectional: [W1,b1] ... [W_{N+1},b_{N+1}] [Wt,dummy].
 * numTemporal = k > 1: [W1,b1] ... [W_{N+1},b_{N+1}] then, per temporal layer in ascending order,
 * [Wtf_j,dummy] [Wtb_j,dummy] (unidirectional: [Wt_j,dummy]); for k = 1 this is the layout above.
 * layerNorm = 1 appends [gamma_i, beta_i] of every normalised hidden layer i, in ascending i.
 * peephole = 1 then appends [P_f,j, dummy] [P_b,j, dummy] (unidirectional: [P_j, dummy]) of every temporal layer j in
 * ascending order, each P 3 x H.
 * selfCondition = 1 then appends [W_c, b_c], W_c layerSize x outputDim and b_c layerSize x 1, behind everything else;
 * like [gamma, beta] and P they lie behind the range L2 regularisation and weight noise see. */
/* maskFeatDim = nu > 0 adds no parameter, and neither do weightNoise = 1, zoneout = 1 and interLayer > 0. */
int64_t ctcb_brnn_param_count(const ctcb_brnn_config *cfg);
int ctcb_brnn_num_tensors(const ctcb_brnn_config *cfg);                    /* 2 * len(stack) */
int ctcb_brnn_tensor_info(const ctcb_brnn_config *cfg, int idx, int64_t *offset, int32_t *rows, int32_t *cols);
/* numTemporal = k > 1 adds k * (2 bi-directional / 1 uni-directional) buffers of maxT*maxB*layerSize floats, each
 * rounded up to 256 bytes, to the one-layer size: For_j (and Back_j) of every temporal layer above the first, and a
 * second dFor / dBack pair that consecutive layers alternate with.
 * cell = 1 (R = maxT*maxB, every buffer rounded up to 256 bytes): an LSTM layer's X_i is G wide instead of H, its D_i
 * max(H, outputDim, G) wide; per LSTM layer c of each direction and, bi-directional, the output For + Back (R*H
 * each); the two column-sum areas grow to G wide, the sweep scratch holds 2*maxB*H floats, and the split-K areas
 * are sized for the G-row contractions and the 4H x H recurrent weight gradients.
 * layerNorm = 1 appends, behind everything else: per normalised layer z (R*H floats) and the row statistics mu and
 * rstd (R floats each), then ctcb_layernorm_workspace_bytes(R, H) for the parameter-gradient partials.  The forward
 * workspace (ctcb_brnn_forward_workspace_bytes) does not grow: a forward-only call normalises in place.
 * subsample = k >= 2 sizes every buffer that only maps >= L use (X_i, D_i, For / Back, c, the LSTM output, z / mu /
 * rstd, the CTC area at Tmax') for R' = ceil(maxT / k) * maxB rows; the dFor / dBack pairs, the split-K, column-sum and
 * layer-norm partial areas for their largest user; and appends, behind everything else, S and dS (R' * k * n floats
 * each, n the width of layer L - 1) and T' (maxB int32).  The forward workspace sizes its slabs, For / Back and c
 * from the rows of the maps that use them in the same way and appends S and T', so it stays within the training
 * workspace.  With k <= 1 no offset moves and nothing is appended.
 * peephole = 1 (with a temporal layer) appends, behind everything else, the partial sums of the peephole weight
 * gradients, ctcb_lstm_peephole_grad_workspace_bytes(Tmax_l, maxB, layerSize, ndir) bytes for the frames Tmax_l of the
 * lowest temporal layer (maxT, or ceil(maxT / k) above the subsampling point).  The forward workspace does not grow.
 * maskFeatDim = nu > 0 appends, behind everything else, the masked copy of a call's features: maxT*maxB*inputDim floats
 * rounded up to 256 bytes.  No other offset moves, and the forward workspace does not grow.
 * weightNoise = 1 appends, behind everything else, the noisy copy of the parameters: ctcb_brnn_param_count floats
 * rounded up to 256 bytes.  No other offset moves, and the forward workspace does not grow.
 * zoneout = 1 (with a temporal layer) appends, behind everything else, the BPTT sweep's dh carry: 2*maxB*layerSize
 * floats rounded up to 256 bytes.  No other offset moves, and the forward workspace does not grow.
 * interLayer = m >= 1 appends, behind everything else, with R_m = T_m maxB (T_m = maxT, or ceil(maxT / k) when
 * m >= subsampleLayer), each area rounded up to 256 bytes: A and D_aux (R_m * outputDim floats each), the intermediate
 * nll (maxB floats) and skips (maxB int32), and, only where the intermediate CTC runs on more frames than the main one
 * (m < subsampleLayer with k >= 2), its own CTC area of ctcb_ctc_workspace_bytes(maxB, maxT, maxLabels) bytes; otherwise
 * it shares the main CTC's area.  No other offset moves, and the forward workspace does not grow.
 * selfCondition = 1 appends, behind those, X'_m (R_m * layerSize floats), P and dA (R_m * outputDim floats each), each
 * rounded up to 256 bytes.  No other offset moves, except that with weightNoise = 1 the noisy copy holds W_c and b_c
 * too (it is ctcb_brnn_param_count floats) and what lies behind it moves by as much.  The forward workspace appends A and P (R_m * outputDim floats each,
 * rounded up to 256 bytes), and its split-K area also covers the A and conditioning contractions at every R <= R_m
 * (within the training area), so that they take the plans of a training call. */
size_t ctcb_brnn_workspace_bytes(const ctcb_brnn_config *cfg);
/* Byte offset, inside the workspace, of a uint32 that the recurrent-sweep kernels set non-zero when an
 * inter-CTA wait timed out (results are then invalid; never a hang).  Callers that synchronise anyway
 * (e.g. for the per-step log line) should read it.  The value names the kernel whose wait timed out:
 * 1 the generic sweep, 2 the cluster sweep, 3 the tensor-core sweep, 4 the LSTM sweep. */
size_t ctcb_brnn_error_flag_offset(const ctcb_brnn_config *cfg);
/* Workspace of a forward-only call (grads == NULL): two ping-pong activation slabs, For and Back (For only when
 * unidirectional, neither without a temporal layer), the split-K area of the forward contractions, the sweep
 * scratch and counters -- no CTC, delta or weight-gradient buffers.  *error_flag_offset (may be NULL) receives the
 * byte offset of the sweep error flag inside it (same meaning as ctcb_brnn_error_flag_offset).  0 for an invalid
 * config.  A forward-only call always uses this layout, in any workspace of at least this size (the training size
 * included), and launches the same kernels with the same plans as a training call of the same B and Tmax, so its
 * probs_out is bit-identical to that call's -- except under zoneout probabilities > 0, where a forward-only call runs
 * the expectation cell and a training call the drawn masks (zoneout, above). */
size_t ctcb_brnn_forward_workspace_bytes(const ctcb_brnn_config *cfg, size_t *error_flag_offset);

/* Diagnostic hook (used by the parity tests): byte offset inside the workspace of the activations the LAST
 * ctcb_brnn_cost_and_grad TRAINING call (grads != NULL) left behind, time-major [Tmax][B][*width] with that call's
 * B and Tmax; a forward-only call lays its buffers out differently (ctcb_brnn_forward_workspace_bytes).
 * what = 0: output of affine map `layer` (1..numLayers+1; For+Back at the temporal layer, logits at the last),
 * what = 1 / 2: For / Back of the temporal layer (brnnet.py:143-153).  With numTemporal > 1, `layer` names which
 * temporal layer (temporalLayer .. temporalLayer+k-1; Back exists only when bi-directional); with one temporal
 * layer it is ignored.  With dropout on (ctcb_brnn_set_dropout), the ReLU hidden layers' entries hold the dropped and
 * rescaled activations.  cell = 1 only: what = 3 the activated gates (G wide, the same buffer as what = 0 of that layer),
 * 4 / 5 c of the forward / backward direction (H wide).  subsample = k >= 2: the entries of maps >= L (and of their
 * temporal layers) are [Tmax'][B][width] with that call's Tmax' = ceil(Tmax / k); what = 6 is S, the stacked input of
 * map L, [Tmax'][B][k n] (`layer` is ignored).  what = 7 is the delta of affine map `layer` (1..numLayers+1), the
 * buffer that map's weight and bias gradients read, [T][B][rows] with rows its output width (G at an LSTM layer):
 * dz after layer normalisation, the gate gradients at an LSTM layer, the BPTT result at a uni-directional clipped-ReLU
 * temporal layer.  CTCB_EINVAL where a later stage of the call overwrites it: a uni-directional clipped-ReLU temporal
 * layer above the lowest two of its stack.  interLayer = m >= 1 only (`layer` is ignored): what = 8 the intermediate
 * logits A, 9 D_aux = lambda d(nll_aux)/dA (both [T_m][B][outputDim]), 10 the intermediate nll (float32[B]), 11 its
 * skips (int32[B]).  selfCondition = 1 only (`layer` is ignored): what = 12 X'_m (layerSize wide), 13 P, 14 dA (both
 * outputDim wide), all [T_m][B][width].  A layer-normalised hidden layer `layer` only: what = 15 its z, the
 * contraction's output before the normalisation (layerSize wide), 16 / 17 its row statistics Mu / Rstd (width 1), all
 * [T][B][width] at that layer's rate.  maskFeatDim > 0 only (`layer` is ignored): what = 18 the masked copy of the
 * features that every stage of a call with input masks on reads, [Tmax][B][inputDim].  weightNoise = 1 only (`layer`
 * is ignored): what = 19 the noisy copy of the flat parameter vector that every stage of a call with noise on reads,
 * *width = ctcb_brnn_param_count floats.  Each of 15..19 is CTCB_EINVAL where its feature is off. */
int ctcb_brnn_activation_offset(const ctcb_brnn_config *cfg, int what, int layer, size_t *offset, int32_t *width);

/* With temporal layers, refuses (CTCB_EINVAL, with the planner's message) a config whose recurrent sweep the device
 * cannot hold at maxB: the LSTM sweep (above), or for cell = 0 the plan ctcb_debug_sweep_plan(layerSize, maxB, ndir)
 * reports, whose tensor-core plan shrinks with the batch and whose generic plan needs ndir * ceil(H / 32) co-resident
 * CTAs at any batch.  Without a device nothing is checked. */
int ctcb_brnn_create(const ctcb_brnn_config *cfg, ctcb_brnn **out);
void ctcb_brnn_destroy(ctcb_brnn *h);

/* costAndGrad over a batch (brnnet.py:117-249 per utterance; gradients SUMMED over utterances).
 * feats     : time-major [Tmax][B][inputDim] fp32 (frame (t,u) contiguous)
 * params    : flat parameter vector; grads: same layout, overwritten
 * cost_out  : float32[B] per-utterance nll (L2 term is returned separately in *regcost_out, device float)
 * probs_out : optional [Tmax][B][outputDim] softmax output (forward-only mode when grads==NULL,
 *             brnnet.py:171-173; that mode needs only ctcb_brnn_forward_workspace_bytes of workspace)
 * stats_out : optional device float[4] = {number of non-skipped utterances, sum of their nll,
 *             number skipped, sweep error flag (see ctcb_brnn_error_flag_offset)}.  Callers place it directly behind the flat gradient so that the
 *             data-parallel all-reduce of the gradient carries it along.  With interLayer > 0 it is float[6]: those
 *             four, then the sum of the intermediate nll over the utterances its CTC kept and the number it skipped,
 *             summed over micro-batches and ranks as the first four are.
 */
int ctcb_brnn_cost_and_grad(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt,
                            const int32_t *labels, const int32_t *label_off, int B, int Tmax,
                            const float *params, float *grads, float *cost_out, int32_t *skip_out,
                            float *regcost_out, float *probs_out, float *stats_out,
                            void *workspace, size_t ws_bytes, void *stream);

/* Gradient accumulation: one step computed as several calls, each on a micro-batch of at most maxB utterances
 * (gradients SUMMED over all of them, so the result equals one call on the whole step up to fp32 summation order).
 * Same arguments as ctcb_brnn_cost_and_grad plus `flags`:
 *   CTCB_PART_FIRST : overwrite every gradient tensor and stats_out (their earlier contents are ignored, NaN
 *                     included; the alignment gaps between tensors of the flat vector are never written);
 *                     without it every gradient tensor and the statistics tail are ADDED into (the error flag
 *                     only grows, so it stays non-zero once any micro-batch set it);
 *   CTCB_PART_LAST  : finish the step: the data-parallel exchange (ctcb_brnn_set_comm), the reg*W gradient
 *                     (unless deferred, ctcb_brnn_set_deferred_l2) and *regcost_out, each once per step; other
 *                     calls leave regcost_out untouched.
 * cost_out / skip_out are per call (pass pointers offset to the micro-batch's utterances).  Every rank of a
 * data-parallel step must make exactly one LAST call (or ctcb_brnn_exchange_only); it may make any number of
 * calls before it.  ctcb_brnn_cost_and_grad == ctcb_brnn_cost_and_grad_part(..., CTCB_PART_FIRST | CTCB_PART_LAST). */
#define CTCB_PART_FIRST 1
#define CTCB_PART_LAST 2
int ctcb_brnn_cost_and_grad_part(ctcb_brnn *h, const float *feats, const int32_t *T_per_utt,
                                 const int32_t *labels, const int32_t *label_off, int B, int Tmax,
                                 const float *params, float *grads, float *cost_out, int32_t *skip_out,
                                 float *regcost_out, float *probs_out, float *stats_out, int flags,
                                 void *workspace, size_t ws_bytes, void *stream);

/* L2 regularisation under data parallelism.  By default ctcb_brnn_cost_and_grad adds reg*W to the weight
 * gradients itself (brnnet.py:197-198,244-247).  A data-parallel caller SUMS the gradient over ranks and must
 * add reg*W exactly once: it switches the handle to deferred mode (the call then only reports the L2 cost) and
 * calls ctcb_brnn_apply_l2_f32 on the reduced gradient. */
int ctcb_brnn_set_deferred_l2(ctcb_brnn *h, int deferred);
int ctcb_brnn_apply_l2_f32(ctcb_brnn *h, const float *params, float *grads, void *stream);

/* ---- inverted dropout on the ReLU hidden layers (not in the reference) ----------------------------------------
 * When p > 0, every TRAINING call (grads != NULL) masks the output X_i of each hidden layer i (1..numLayers) that is
 * not temporal, in place, right after its forward contraction: the input, the temporal layers' outputs and the logits
 * are never dropped, and forward-only calls (grads == NULL) never drop.  The mask is a pure function of
 * (seed, step, i, g, t, j) -- g the utterance's index in the step's whole minibatch, t the frame, j the unit:
 *     r = Philox4x32-10(counter = (step mod 2^32, g mod 2^32, t, (i << 24) | (j / 4)),
 *                       key = (seed mod 2^32, seed >> 32))[j % 4]       (curand_Philox4x32_10, one call per 4 units)
 *     keep iff r >= thr,  thr = floor(p * 2^32)  (float64);  kept: x * s,  s = float32(1 / (1 - p))  (float64, rounded
 *     once);  dropped: 0.
 * step is the int64 at `step` (DEVICE memory), read by every training call when it runs, so a captured CUDA graph
 * draws the mask of the counter's current value; the handle owns no memory, the caller owns the counter.  The delta
 * contraction of layer i runs with alpha = s and the ReLU mask X_i > 0 (which removes the dropped units), so the
 * gradient is that of the dropped net.  The activation hook (ctcb_brnn_activation_offset) returns the dropped X_i.
 * p == 0 (the default) disables it: a training call then issues exactly the launches and bits it does without.
 * CTCB_EINVAL for p < 0, p >= 1, NaN, or p > 0 with a null step.  Host-only: no device work. */
int ctcb_brnn_set_dropout(ctcb_brnn *h, float p, uint64_t seed, const int64_t *step);
/* Utterance u of the following calls is minibatch utterance g = first + stride * u: rank + world * (u0 + u) for rank
 * `rank` of `world` (round-robin shards) and a micro-batch starting at position u0 of the rank's shard, so one call, a
 * micro-batched step and a data-parallel step draw the same mask for the same utterance.  The same g places the
 * utterance for the input masks (ctcb_brnn_set_input_masks).  Default (0, 1).  CTCB_EINVAL for first < 0 or
 * stride < 1.  Host-only. */
int ctcb_brnn_set_dropout_utts(ctcb_brnn *h, int64_t first, int64_t stride);
/* *step += 1 on `stream` (one thread); inside a capture it becomes part of the graph like any other launch.  The
 * counter is the optimisation step: the dropout mask, the adaptive optimisers (ctcb_adagrad_step_f32,
 * ctcb_adam_step_f32) and the weight average (ctcb_ema_update_f32) read the same one, and sgd.SGD advances it once per
 * step, so it equals SGD.it. */
int ctcb_dropout_advance(int64_t *step, void *stream);

/* ---- SpecAugment: frequency and time masks of the input features (Park et al., Interspeech 2019) --------------------
 * Layout (maskFeatDim = nu > 0): row t' of utterance u holds c = inputDim / nu frame slots of nu bins each, frame-major
 * (Kaldi splice-feats), c odd, h = (c - 1) / 2; slot j holds raw frame clamp(t' + j - h, 0, T_u - 1), so splicing
 * repeats the edge frames.  c = 1 is features without splicing.
 * Policy: m_F = freqMasks, F = freqWidth, m_T = timeMasks, T = timeWidth, p = timeRatio.  Minibatch utterance g (as
 * ctcb_brnn_set_dropout_utts places it) at optimisation step s draws, for mask k = 0 .. m_F + m_T - 1, one block
 *     (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32, g mod 2^32, 0, k), key = (seed mod 2^32, seed >> 32))
 * (k < 2^24, dropout's fourth counter word is >= 2^24, so the two can share a seed), and with 64-bit integer products:
 *   k <  m_F: width w = (r0 (F + 1)) >> 32, start f0 = (r1 (nu - w + 1)) >> 32: bins [f0, f0 + w) are masked;
 *   k >= m_F: W = min(T, floor(p T_u)) (the product in float64), w = (r0 (W + 1)) >> 32, t0 = (r1 (T_u - w + 1)) >> 32:
 *             raw frames [t0, t0 + w) are masked.
 * Element (t' < T_u, slot j, bin b) becomes +0.0 where b lies in a frequency band or its raw frame in a time band
 * (bands may overlap); every other element, the padding rows t' >= T_u included, is copied bit for bit.
 * Limits: m_F and m_T in 0..64, 0 <= F <= nu, T >= 0, p in [0, 1].
 *
 * ctcb_brnn_set_input_masks: every TRAINING call (grads != NULL) then writes the masked copy of feats into its workspace
 * (maxT*maxB*inputDim floats behind everything else) with one pass on the main chain, and every stage reads that copy:
 * map 1's contraction, the frame stacking when subsampleLayer = 1, map 1's weight gradient.  feats is never written, so
 * a replayed step over one device batch does not mask twice and forward-only calls (grads == NULL, which never mask)
 * see the original features.  step is the int64 DEVICE counter of ctcb_dropout_advance, read when the pass runs.  Both
 * counts 0 (the default) disables it: the call reads feats and issues exactly the launches it does without.
 * CTCB_EINVAL for values outside the limits, counts > 0 on a config with maskFeatDim = 0, or counts > 0 with a null
 * step.  Host-only: no device work. */
int ctcb_brnn_set_input_masks(ctcb_brnn *h, int freqMasks, int freqWidth, int timeMasks, int timeWidth,
                              double timeRatio, uint64_t seed, const int64_t *step);
/* The pass on its own, with the launch a training call makes: out = feats masked for the utterances g = first +
 * stride * u, both [Tmax][B][inputDim] (out must not overlap feats), T_per_utt int32[B] (<= Tmax).  16-byte accesses
 * where inputDim % 4 == 0 and both arrays are 16-byte aligned, else 4-byte ones.  With both counts 0 it copies and step
 * may be NULL.  CTCB_EINVAL for a layout the config would refuse, a policy outside the limits, first < 0, stride < 1,
 * B or Tmax < 1, or B * Tmax >= 2^31. */
int ctcb_input_mask_f32(const float *feats, const int32_t *T_per_utt, int B, int Tmax, int inputDim, int featDim,
                        int freqMasks, int freqWidth, int timeMasks, int timeWidth, double timeRatio, uint64_t seed,
                        const int64_t *step, int64_t first, int64_t stride, float *out, void *stream);

/* ---- Gaussian weight noise (Graves, Mohamed & Hinton, ICASSP 2013; Graves & Jaitly, ICML 2014) -----------------------
 * Noised tensors: the ones L2 regularisation sees, the even tensors 0 .. nreg - 1 of the flat vector -- W of every
 * affine map and every recurrent matrix (the clipped-ReLU Wtf / Wtb / Wt, the LSTM U).  Biases, the dummies, the
 * layer-norm [gamma, beta] and the peephole P are used as they are.
 * Draw: at optimisation step s, element e of a noised matrix (e its offset in the flat vector; every tensor is 16-byte
 * aligned, so the quad q = e / 4 never straddles two tensors), j = e % 4:
 *     (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32, q mod 2^32, 1, 0), key = (seed mod 2^32, seed >> 32))
 *     (a, b) = (r0, r1) for j in {0, 1}, (r2, r3) for j in {2, 3}
 *     u1 = (a + 1) 2^-32,  u2 = b 2^-32,  rho = sqrt(-2 ln u1)                 (float64)
 *     z = rho cos(2 pi u2) for even j, rho sin(2 pi u2) for odd j              (float64)
 *     w' = w + float32(sigma z)                                                (sigma z rounded once, a float32 add)
 * Every other element, the alignment gaps included, is copied bit for bit.  The three draws of a seed never meet:
 * dropout's fourth counter word is (layer << 24) | .. >= 2^24, SpecAugment's third word is 0, this rule's third word
 * is 1 and its fourth 0.
 * One draw per step: the noise does not depend on the utterance, the rank or the micro-batch, so a batch of B
 * utterances shares one noisy net (at one utterance per step, the reference's schedule, that is noise per sequence).
 *
 * ctcb_brnn_set_weight_noise: with sigma > 0 every TRAINING call (grads != NULL) writes w' into its workspace (behind
 * everything else, with weightNoise = 1) with one pass at the start of the main chain, and every stage that reads a
 * weight reads that copy: the forward contractions, the recurrent sweeps, the delta contractions.  The gradient is
 * that of the returned cost, evaluated at w'.  The L2 term (reg w in the gradient, reg/2 |w|^2 in regcost) and the
 * data-parallel exchange see the CLEAN params, and params is never written, so an update applies to the clean w (with
 * Nesterov the noise sits on the look-ahead point the caller passes).  Every training call forms the copy from params,
 * so the micro-batches of one step see the same bits.  step is the int64 DEVICE counter of ctcb_dropout_advance, read
 * when the pass runs.  Forward-only calls (grads == NULL) never add noise.  sigma = 0 (the default) disables it: the
 * call reads params and issues exactly the launches it does without.  CTCB_EINVAL for sigma negative, NaN or
 * infinite, sigma > 0 on a config with weightNoise = 0, or sigma > 0 with a null step.  Host-only: no device work. */
int ctcb_brnn_set_weight_noise(ctcb_brnn *h, float sigma, uint64_t seed, const int64_t *step);
/* The pass on its own, with the launch a training call makes under the handle's settings: out = params with the
 * noise of the current step (ctcb_brnn_param_count floats each; out must not overlap params).  With sigma = 0 it
 * copies.  16-byte accesses where both are 16-byte aligned, else 4-byte ones. */
int ctcb_brnn_weight_noise_f32(ctcb_brnn *h, const float *params, float *out, void *stream);

/* ---- zoneout of the LSTM cell's state (zoneout = 1, above) ----------------------------------------------------------
 * ctcb_brnn_set_zoneout: zc and zh are the probabilities z_c and z_h of every LSTM layer; training calls draw the masks
 * with seed and the int64 DEVICE counter step (ctcb_dropout_advance's), read when each sweep runs, so the micro-batches
 * of one step, its shards (ctcb_brnn_set_dropout_utts) and a replayed graph draw the same masks.  Forward-only calls use
 * the expectation.  zc = zh = 0 (the default) disables it: every call issues exactly the launches and bits it does
 * without.  CTCB_EINVAL for a value outside [0, 1) (NaN included), or a value > 0 on a config with zoneout = 0.  step
 * may be NULL for forward-only use; a training call with a value > 0 and a NULL step then returns CTCB_EINVAL before it
 * launches anything.  Host-only: no device work. */
int ctcb_brnn_set_zoneout(ctcb_brnn *h, float zc, float zh, uint64_t seed, const int64_t *step);

/* ---- layer normalisation on its own (layerNorm = 1, above) -----------------------------------------------------
 * Rows are [R][H] fp32, 1 <= H <= CTCB_LAYERNORM_MAX_H; with H % 4 == 0 every pointer must be 16-byte aligned.
 * forward : y = relu(gamma (z - mu) rstd + beta) per row; y may alias z; mu / rstd (R floats each) receive the row
 *           statistics, or are both NULL.  The same device code writes y either way, so the bits of y do not depend on it.
 * backward: delta holds g on entry and dz on return (in place); z, mu, rstd as the forward left them; dgamma / dbeta
 *           (H floats each) receive the sums over the rows, or, with accumulate != 0, have them added.  workspace:
 *           ctcb_layernorm_workspace_bytes(R, H) bytes (per-CTA partial sums, added in a fixed order: the bits depend
 *           only on R, H and the inputs).  0 for H out of range. */
size_t ctcb_layernorm_workspace_bytes(int64_t R, int H);
int ctcb_layernorm_forward_f32(const float *z, float *y, float *mu, float *rstd, const float *gamma, const float *beta,
                               int64_t R, int H, void *stream);
int ctcb_layernorm_backward_f32(float *delta, const float *z, const float *mu, const float *rstd, const float *gamma,
                                float *dgamma, float *dbeta, int64_t R, int H, int accumulate, void *workspace,
                                size_t ws_bytes, void *stream);

/* ---- the training step's reductions on their own: the launches a training call makes ----------------------------
 * colsum : out[j] = sum over the R rows of the row-major R x n matrix delta (the bias gradients), or with accumulate
 *          != 0 added into out.  workspace: 16-byte aligned, ctcb_colsum_workspace_bytes(R, n) bytes of partial sums
 *          (CTCB_ENOMEM when shorter); 0 for R or n < 1.  Stage 1 sums row blocks in a fixed order, stage 2 adds the
 *          blocks' partials in order, so the bits depend only on R, n, the inputs, the alignment of delta and the
 *          device's SM count.  CTCB_EINVAL for R or n < 1, or more than 65535 row blocks of 128.
 * ctcb_debug_colsum_plan: out (HOST, 4 int32) = {path: 1 wide (n % 4 == 0 and delta 16-byte aligned: each thread a
 *          float4 column group, 4 rows per loop step) / 0 narrow (8 strided threads per column), column blocks,
 *          rows per block (wide: R / (2 SMs / column blocks) within [128, 1024]; narrow: 1024), row blocks}.
 * softmax_rows: p = softmax of each row of the row-major R x K matrix x, the forward-only probabilities of a
 *          ctcb_brnn_cost_and_grad call (probs_out); one warp per row.
 * softmax_rows_backward: out = p (dp - sum_k p_k dp_k) + add per row of the row-major R x K matrices, the gradient of a
 *          row softmax p with respect to its logits given dp = dL/dp, plus add (may be NULL); out may alias dp.  The
 *          dA of self-conditioned CTC (selfCondition, above); one warp per row.  Argument checks as softmax_rows. */
size_t ctcb_colsum_workspace_bytes(int64_t R, int n);
int ctcb_colsum_f32(const float *delta, int64_t R, int n, float *out, int accumulate, void *workspace, size_t ws_bytes,
                    void *stream);
int ctcb_debug_colsum_plan(int64_t R, int n, const float *delta, int32_t *out);
int ctcb_softmax_rows_f32(const float *x, float *p, int64_t R, int K, void *stream);
int ctcb_softmax_rows_backward_f32(const float *p, const float *dp, const float *add, float *out, int64_t R, int K,
                                   void *stream);

/* ---- frame stacking on its own (subsample = k, above) ----------------------------------------------------------
 * x / d_out are time-major [Tmax][B][n], s_out / ds [ceil(Tmax / k)][B][k n], T_per_utt int32[B] (<= Tmax).
 * stack  : s_out[t'][u][m n + j] = x[k t' + m][u][j], 0 where k t' + m >= T_u; lens_out (int32[B], may be NULL)
 *          receives ceil(T_u / k).
 * unstack: d_out[t][u][j] = ds[t / k][u][(t % k) n + j] for t < T_u, 0 beyond.
 * Exact copies: 16-byte accesses where n % 4 == 0 and both arrays are 16-byte aligned, else 4-byte ones. */
int ctcb_frame_stack_f32(const float *x, const int32_t *T_per_utt, int Tmax, int B, int n, int k, float *s_out,
                         int32_t *lens_out, void *stream);
int ctcb_frame_unstack_f32(const float *ds, const int32_t *T_per_utt, int Tmax, int B, int n, int k, float *d_out,
                           void *stream);

/* ---- the time recurrences of the temporal layer on their own (replaces the per-frame loops
 *      brnnet.py:144-152 [mode 0] and brnnet.py:208-224 [mode 1]) -------------------------------
 * All arrays time-major [T][B][H] fp32.  mode 0: outF[t] = clip(pre[t] + outF[t-1].Wf^T, 0, maxAct),
 * outB mirrored in time with Wb; utterance u is zero beyond T_per_utt[u].
 * mode 1: outF[t] = within(actF[t]) * (pre[t] + outF[t+1].Wf), outB mirrored.
 * Wb == NULL (with outB/actB ignored) runs the forward-in-time direction alone: the uni-directional layer of
 * nnets/rnnet.py:112-116 [mode 0] and :162-177 [mode 1].
 * scratch: 256-byte aligned device memory, >= 4096 bytes (word 0 = error flag, cleared by the call); the tensor-core
 * kernel (H >= 1024, sweep_tc.cu) additionally needs room for the (hi, lo) stacks of the recurrent matrices and the
 * ring of state low halves: ctcb_brnn_sweep_workspace_bytes(H, B) in total; where that kernel applies
 * (ctcb_sweep_uses_tensor_cores) a smaller scratch is an error (CTCB_ENOMEM), never a slower kernel. */
size_t ctcb_brnn_sweep_workspace_bytes(int H, int B);
int ctcb_brnn_sweep_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, const float *pre,
                        const float *Wf, const float *Wb, float *outF, float *outB, const float *actF,
                        const float *actB, float maxAct, void *scratch, size_t scratch_bytes, void *stream);
/* The same in TF32 mode (ctcb_brnn_config.tf32, above), same arguments and scratch: the tensor-core kernel rounds W
 * (W^T) and each step's state to TF32 and runs one MMA per product; S_t itself stays the exact fp32 output of the
 * step.  The cluster and generic kernels run as ctcb_brnn_sweep_f32, with its bits. */
int ctcb_brnn_sweep_tf32(int mode, int T, int B, int H, const int32_t *T_per_utt, const float *pre,
                         const float *Wf, const float *Wb, float *outF, float *outB, const float *actF,
                         const float *actB, float maxAct, void *scratch, size_t scratch_bytes, void *stream);
/* The LSTM recurrences of one temporal layer on their own (cell = 1).  Time-major arrays; G = 8H with Ub, 4H without.
 * mode 0: gates [T][B][G] holds pre = W x + b on entry and the activated gates i, f, g, o (0 at padded frames) on
 *   return; hF / hB [T][B][H] receive h, cF / cB [T][B][H] receive c.
 * mode 1: gates, cF / cB as mode 0 left them, dh [T][B][H] the gradient w.r.t. the layer's output (the same for both
 *   directions); dz [T][B][G] receives the gate gradients of both directions (hF / hB are not read).
 * Ub == NULL runs the forward-in-time direction alone.  scratch: 256-byte aligned, ctcb_lstm_sweep_workspace_bytes(H,
 * B) bytes (word 0 = error flag, cleared by the call and set when a wait between CTAs timed out; the dc carry). */
size_t ctcb_lstm_sweep_workspace_bytes(int H, int B);
int ctcb_lstm_sweep_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates, const float *Uf,
                        const float *Ub, float *hF, float *hB, float *cF, float *cB, const float *dh, float *dz,
                        void *scratch, size_t scratch_bytes, void *stream);
/* The same with peephole connections (peephole = 1, above): Pf / Pb the [3][H] peephole vectors (rows i, f, o) of the
 * two directions; Pb is ignored when Ub == NULL.  Same scratch; mode 1 carries the whole dc_{t+1} term of dc_t in it. */
int ctcb_lstm_sweep_peephole_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates, const float *Uf,
                                 const float *Ub, const float *Pf, const float *Pb, float *hF, float *hB, float *cF,
                                 float *cB, const float *dh, float *dz, void *scratch, size_t scratch_bytes, void *stream);
/* The same with zoneout (zoneout = 1, above), with peephole connections when Pf != NULL.  train != 0 draws the masks of
 * (seed, *step, g = first + stride * b, t, layer, direction, j), train == 0 uses the expectation; mode 1 runs the BPTT
 * above with those lambdas (with train == 0, lambda = z).  hF / hB are read in mode 0 (h_{t-1}).  The BPTT carries
 * lambda_h dh in a second [ndir][B][H] area: scratch is ctcb_lstm_sweep_zoneout_workspace_bytes(H, B) bytes.
 * CTCB_EINVAL for zc or zh outside [0, 1), train with a NULL step, first < 0, stride < 1 or layer outside 1..255. */
size_t ctcb_lstm_sweep_zoneout_workspace_bytes(int H, int B);
int ctcb_lstm_sweep_zoneout_f32(int mode, int T, int B, int H, const int32_t *T_per_utt, float *gates, const float *Uf,
                                const float *Ub, const float *Pf, const float *Pb, float *hF, float *hB, float *cF,
                                float *cB, const float *dh, float *dz, float zc, float zh, int train, uint64_t seed,
                                const int64_t *step, int64_t first, int64_t stride, int layer, void *scratch,
                                size_t scratch_bytes, void *stream);
/* The peephole weight gradients of one LSTM layer: dz [T][B][G] as mode 1 of the sweep wrote it, cF / cB [T][B][H] as
 * mode 0 did (cB == NULL: one direction, G = 4H, dPb ignored); dPf / dPb [3][H] receive dp_i, dp_f, dp_o, or with
 * accumulate != 0 have them added.  workspace: ctcb_lstm_peephole_grad_workspace_bytes(T, B, H, ndir) bytes of partial
 * sums over fixed chunks of rows, added in a fixed order: the bits depend only on T, B, H and the inputs. */
size_t ctcb_lstm_peephole_grad_workspace_bytes(int T, int B, int H, int ndir);
int ctcb_lstm_peephole_grad_f32(int T, int B, int H, const float *dz, const float *cF, const float *cB, float *dPf,
                                float *dPb, int accumulate, void *workspace, size_t ws_bytes, void *stream);
/* The LSTM sweep's plan for (H, B, ndir) of the kernel that runs, without (peephole = 0) or with peephole connections,
 * under the knobs in effect (INTEGRATION.md section 4: CTCB_LSTM, CTCB_LSTM_PARTS): out (HOST, 4 int32) = {KI (H / 32
 * with U in registers, else 0), utterance partitions, CTAs of that kernel per SM, 8-utterance tiles per partition (the
 * last partitions may get fewer, or none)}; or the error the sweep call and ctcb_brnn_create return for a width, or a
 * forced partition count, the device cannot hold. */
int ctcb_debug_lstm_plan(int H, int B, int ndir, int peephole, int32_t *out);
/* The same for the zoneout kernels (ctcb_lstm_sweep_zoneout_f32), whose occupancy is their own. */
int ctcb_debug_lstm_zoneout_plan(int H, int B, int ndir, int peephole, int32_t *out);
/* 1 when the recurrences of a (layerSize H, B utterances, bi-directional) step run on the tensor-core kernel. */
int ctcb_sweep_uses_tensor_cores(int H, int B);
/* The plan ctcb_brnn_sweep_f32 launches for (H, B, ndir = 2 bi-directional / 1 forward in time only) on the current
 * device, under the knobs in effect (INTEGRATION.md section 4: CTCB_SWEEP*).  out (HOST, 8 int32):
 *   {kernel: 0 generic / 1 cluster / 2 tensor-core, KI (H / 32 with register-resident weights, else 0),
 *    CS (tensor-core: K-slices per cluster; cluster: CTAs per cluster; generic: 0),
 *    NB (cluster: utterances per cluster) or NS (tensor-core: utterance splits) or the generic kernel's partitions,
 *    NP (tensor-core: utterances per split), ring stages, partial_own (tensor-core: 1 when the split-K partial has its
 *    own shared memory), CTAs of the generic kernel per SM (other kernels: 0)}.
 * Returns the error the launch itself, and ctcb_brnn_create for a ReLU net of that width at maxB, would return for a
 * plan the device cannot hold: CTCB_EINVAL for a width whose shared memory or co-resident CTAs exceed the device, or a
 * forced partition count it cannot hold co-resident. */
int ctcb_debug_sweep_plan(int H, int B, int ndir, int32_t *out);
/* The plan ctcb_brnn_sweep_tf32 launches, in the same form. */
int ctcb_debug_sweep_plan_tf32(int H, int B, int ndir, int32_t *out);

/* ---- optimiser (replaces sgd.SGD.run arithmetic, ctc_fast/sgd.py:91-161, and
 *      NNet.updateParams, brnnet.py:251-256) --------------------------------------------------- */
/* w += scale * u over n floats (updateParams) */
int ctcb_axpy_f32(float *w, const float *u, float scale, int64_t n, void *stream);
/* gnorm2_out[0] = sum(g^2) (sgd.py:103-107), deterministic two-stage reduction; scratch >= 4 KB (512 doubles) */
int ctcb_sumsq_f32(const float *g, int64_t n, float *gnorm2_out, void *scratch, void *stream);
/* Fused sgd.py:97-100,130-140,161 given w at the look-ahead point w + mom*v:
 *   w -= mom*v;  alph = alpha*min(1, maxGNorm/sqrt(*gnorm2));  v = mom*v - alph*g;  w += v
 * gnorm2 is read on the device (no host sync).  n_valid (optional device float): when it reads 0
 * every utterance of the step was skipped and only the undo `w -= mom*v` is applied, as the
 * reference's `if skip: continue` does (sgd.py:109-111). */
int ctcb_sgd_nesterov_step_f32(float *w, float *v, const float *g, int64_t n, float mom, float alpha,
                               float max_gnorm, const float *gnorm2, const float *n_valid, void *stream);
/* The adaptive rules (not in the reference's working code: its AdaGrad branch, sgd.py:143-158, is never reached).
 * Both run on the step's reduced gradient g (the L2 term already in it), with no look-ahead, clipped as a gradient:
 *   g_c = c*g,  c = min(1, maxGNorm / sqrt(*gnorm2))           (gnorm2 read on the device, as for Nesterov)
 * t is the int64 at `step` (DEVICE memory: the counter of ctcb_dropout_advance), read when the kernel runs; a value
 * below 1 is taken as 1.  When n_valid (optional device float) reads 0, w and every state are left bit for bit
 * unchanged.  Per-step scalars are computed in float64 and rounded to float32 once; the element arithmetic is float32.
 * AdaGrad, state r (the reference's gradt):
 *   gamma_t = 1 - 1/(0.01 t + 1);  r = gamma_t*r + g_c^2;  w -= alpha * g_c / sqrt(r + 1e-10)
 * Adam (Kingma & Ba, Algorithm 1), states m and v:
 *   m = b1*m + (1-b1)*g_c;  v = b2*v + (1-b2)*g_c^2;  w -= alpha * (m/(1-b1^t)) / (sqrt(v/(1-b2^t)) + eps)
 * Checked on the host before any launch: n <= 0 is a no-op; CTCB_EINVAL for a null w, state, g, gnorm2 or step, a
 * non-finite or negative alpha, a beta outside [0, 1), and a non-finite eps or eps <= 0. */
int ctcb_adagrad_step_f32(float *w, float *r, const float *g, int64_t n, float alpha, float max_gnorm,
                          const float *gnorm2, const float *n_valid, const int64_t *step, void *stream);
int ctcb_adam_step_f32(float *w, float *m, float *v, const float *g, int64_t n, float alpha, float beta1,
                       float beta2, float eps, float max_gnorm, const float *gnorm2, const float *n_valid,
                       const int64_t *step, void *stream);
/* Exponential moving average of the weights (Polyak averaging while it warms up), one pass over the flat vector, run
 * after the rule's update on the w it just wrote (Nesterov: the clean weight, the look-ahead undone).  With decay d in
 * [0, 1) and t = max(1, *step), the int64 at `step` (DEVICE memory: the counter of ctcb_dropout_advance) read when the
 * kernel runs:
 *   d_t = min(d, 1 - 1/t)      (float64, rounded to float32 once)
 *   avg = fmaf(d_t, avg - w, w)   element-wise in float32, i.e. avg = w + d_t (avg - w)
 * At t = 1, d_t = 0 and avg becomes a copy of w bit for bit.  While 1 - 1/t < d, avg is the plain mean of the iterates
 * w_1 .. w_t; after that an EMA of decay d (d = 0.9999: the mean of the first 10 000 steps, then the EMA).  When n_valid
 * (optional device float) reads 0, avg is left bit for bit unchanged; the caller still advances the counter.  12 B per
 * parameter.  Checked on the host before any launch: n <= 0 is a no-op; CTCB_EINVAL for a null avg, w or step, and for
 * a decay that is NaN or outside [0, 1). */
int ctcb_ema_update_f32(float *avg, const float *w, int64_t n, float decay, const float *n_valid, const int64_t *step,
                        void *stream);

/* ---- CUDA graphs: replay one optimisation step (the reference issues ~16(N+3)+8(T-1) launches per utterance,
 *      sgd.py:91-161 + brnnet.py:117-249; this library ~40 per minibatch) as ONE graph launch -----------------------
 * Between begin and end, calls into this library on `stream` are captured instead of executed (including the internal
 * side stream and the NCCL exchange); every pointer, size and scalar argument is frozen into the graph, so a graph is
 * valid for one (buffers, B, Tmax, momentum, step size) combination.  Warm the same calls up once before capturing
 * (first-use initialisation is not capturable). */
typedef struct ctcb_graph ctcb_graph;
int ctcb_graph_capture_begin(void *stream);
int ctcb_graph_capture_end(void *stream, ctcb_graph **out);
int ctcb_graph_launch(ctcb_graph *g, void *stream);
void ctcb_graph_destroy(ctcb_graph *g);

/* ---- data-parallel exchange (SURVEY.md 8b/8e; the reference's only device hook is CUDA_DEVICE,
 *      ctc_fast/runNNet.py:117-120, and it has no multi-GPU path) -------------------------------------
 * One process per GPU.  Rank 0 obtains an id (HOST buffer of CTCB_COMM_ID_BYTES) and hands it to the other ranks by
 * whatever channel the host program has (a file, MPI, torch.distributed ...); every rank then creates its
 * communicator with the device it computes on current.  NCCL is loaded at run time (libnccl.so.2). */
#define CTCB_COMM_ID_BYTES 128
typedef struct ctcb_comm ctcb_comm;
int ctcb_comm_get_unique_id(void *id_out /* HOST */);
int ctcb_comm_create(const void *id /* HOST */, int rank, int world, ctcb_comm **out);
void ctcb_comm_destroy(ctcb_comm *comm);
int ctcb_comm_rank(const ctcb_comm *comm);
int ctcb_comm_world(const ctcb_comm *comm);
/* grads[0..n) <- sum over ranks, in place, asynchronous on `stream` (one ncclAllReduce over NVLink). */
int ctcb_allreduce_grads(ctcb_comm *comm, float *grads, int64_t n, void *stream);
/* Attach a communicator to a net: ctcb_brnn_cost_and_grad then performs the exchange itself -- the gradients of the
 * layers at and above the temporal layer are summed over ranks on an internal side stream WHILE the BPTT sweep runs,
 * the remaining tensors and the statistics tail (stats_out, normally grads + param_count) in one grouped launch at
 * the end -- and adds the L2 term once, after the sum.  On return (stream order) `grads` holds the global gradient. */
int ctcb_brnn_set_comm(ctcb_brnn *h, ctcb_comm *comm);
/* For a rank whose shard of the step is empty: the same sequence of collectives on a zero-filled gradient. */
int ctcb_brnn_exchange_only(ctcb_brnn *h, const float *params, float *grads, float *stats_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CTCB200_H */
