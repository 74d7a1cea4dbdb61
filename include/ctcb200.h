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
 *             utterances with unaligned outputs, where the reference returns a wrong loss and gradient)
 * workspace : ctcb_ctc_workspace_bytes(B, Tmax, max_labels) bytes of device scratch.  That size never decreases with B,
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
} ctcb_brnn_config;

typedef struct ctcb_brnn ctcb_brnn; /* opaque; owns no device memory */

/* Flat parameter vector layout: the reference's `stack` order (brnnet.py:38-41,66-72):
 * [W1,b1] ... [W_{N+1},b_{N+1}] [Wtf,dummy] [Wtb,dummy]; W row-major (out x in), dummy = 1 float.
 * unidirectional: [W1,b1] ... [W_{N+1},b_{N+1}] [Wt,dummy].
 * numTemporal = k > 1: [W1,b1] ... [W_{N+1},b_{N+1}] then, per temporal layer in ascending order,
 * [Wtf_j,dummy] [Wtb_j,dummy] (unidirectional: [Wt_j,dummy]); for k = 1 this is the layout above. */
int64_t ctcb_brnn_param_count(const ctcb_brnn_config *cfg);
int ctcb_brnn_num_tensors(const ctcb_brnn_config *cfg);                    /* 2 * len(stack) */
int ctcb_brnn_tensor_info(const ctcb_brnn_config *cfg, int idx, int64_t *offset, int32_t *rows, int32_t *cols);
/* numTemporal = k > 1 adds k * (2 bi-directional / 1 uni-directional) buffers of maxT*maxB*layerSize floats, each
 * rounded up to 256 bytes, to the one-layer size: For_j (and Back_j) of every temporal layer above the first, and a
 * second dFor / dBack pair that consecutive layers alternate with. */
size_t ctcb_brnn_workspace_bytes(const ctcb_brnn_config *cfg);
/* Byte offset, inside the workspace, of a uint32 that the recurrent-sweep kernels set non-zero when an
 * inter-CTA wait timed out (results are then invalid; never a hang).  Callers that synchronise anyway
 * (e.g. for the per-step log line) should read it. */
size_t ctcb_brnn_error_flag_offset(const ctcb_brnn_config *cfg);
/* Workspace of a forward-only call (grads == NULL): two ping-pong activation slabs, For and Back (For only when
 * unidirectional, neither without a temporal layer), the split-K area of the forward contractions, the sweep
 * scratch and counters -- no CTC, delta or weight-gradient buffers.  *error_flag_offset (may be NULL) receives the
 * byte offset of the sweep error flag inside it (same meaning as ctcb_brnn_error_flag_offset).  0 for an invalid
 * config.  A forward-only call always uses this layout, in any workspace of at least this size (the training size
 * included), and launches the same kernels with the same plans as a training call of the same B and Tmax, so its
 * probs_out is bit-identical to that call's. */
size_t ctcb_brnn_forward_workspace_bytes(const ctcb_brnn_config *cfg, size_t *error_flag_offset);

/* Diagnostic hook (used by the parity tests): byte offset inside the workspace of the activations the LAST
 * ctcb_brnn_cost_and_grad TRAINING call (grads != NULL) left behind, time-major [Tmax][B][*width] with that call's
 * B and Tmax; a forward-only call lays its buffers out differently (ctcb_brnn_forward_workspace_bytes).
 * what = 0: output of affine map `layer` (1..numLayers+1; For+Back at the temporal layer, logits at the last),
 * what = 1 / 2: For / Back of the temporal layer (brnnet.py:143-153).  With numTemporal > 1, `layer` names which
 * temporal layer (temporalLayer .. temporalLayer+k-1; Back exists only when bi-directional); with one temporal
 * layer it is ignored. */
int ctcb_brnn_activation_offset(const ctcb_brnn_config *cfg, int what, int layer, size_t *offset, int32_t *width);

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
 *             data-parallel all-reduce of the gradient carries it along.
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
/* 1 when the recurrences of a (layerSize H, B utterances, bi-directional) step run on the tensor-core kernel. */
int ctcb_sweep_uses_tensor_cores(int H, int B);
/* The plan ctcb_brnn_sweep_f32 launches for (H, B, ndir = 2 bi-directional / 1 forward in time only) on the current
 * device, under the knobs in effect (INTEGRATION.md section 4).  out (HOST, 8 int32):
 *   {kernel: 0 generic / 1 cluster / 2 tensor-core, KI (H / 32 with register-resident weights, else 0),
 *    CS (tensor-core: K-slices per cluster; cluster: CTAs per cluster; generic: 0),
 *    NB (cluster: utterances per cluster) or NS (tensor-core: utterance splits) or the generic kernel's partitions,
 *    NP (tensor-core: utterances per split), ring stages, partial_own (tensor-core: 1 when the split-K partial has its
 *    own shared memory), 0}.
 * Returns the error the launch itself would return for a plan the device cannot hold. */
int ctcb_debug_sweep_plan(int H, int B, int ndir, int32_t *out);

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
