"""GPU tests of how the training step (csrc/brnn.cu) wires its kernels together: after one training call with
probabilities, each stage's float32 output, read through ctcb_brnn_activation_offset, against float64 computed from the
step's own float32 inputs, under the element-wise bound of the kernel that stage launched.

Contractions: |C - C64| <= (c0 + c1 L) 2^-24 S (BOUNDS and _chain of test_gemm_plans_gpu.py) at the plan
ctcb_debug_gemm_plan reports for the step's own operand pointers; ReLU is applied to C64, masked entries must be
exactly +0.0.  A second contraction with beta != 0 onto the first's float32 result (the self-conditioning add, the
conditioned delta) takes one bound whose S includes |C0|; where the step adds it onto a buffer that a later stage
overwrites (the intermediate-CTC term before the layer-norm backward), the two together take the sum of both bounds.
Layer norm: C_FWD and the backward bound of test_layernorm_gpu.py from the step's own z, Mu and Rstd; P = softmax(A):
C_SOFTMAX of test_step_reductions_gpu.py; dA: the softmax-backward bound of test_self_cond_gpu.py.

Stages checked, on every net of part (c) of test_step_reductions_gpu.py and on nets with the intermediate CTC,
self-conditioning, weight noise, SpecAugment masks, zoneout and widths that reach the 3xTF32 kernel:
  forward  every map's output the step keeps (X_i, z_i before layer norm, the logits), read from what the map read:
           the masked feature copy, S (an exact stack of layer L - 1), X'_m above the conditioned layer, the noisy
           parameter copy; layer norm and its statistics; dropout (the device's draw, net_oracle.keep_mask: dropped
           entries exactly +0.0, kept ones s y); the
           intermediate logits A, P = softmax(A), X'_m;
  backward every delta of a feed-forward hidden layer against alpha [X_i > 0] (delta_{i+1} W_{i+1}), through the
           unstacking below map L, with alpha D_aux W_{N+1} at interLayer; where the layer-norm backward overwrote g,
           g is recomputed with ctcb_gemm_f32 from the step's own operands at the step's plan (the contraction is
           deterministic per plan, so these are the step's bits), checked, and the backward checked from it; at the
           conditioned layer D'_m and dP the same way, then dA, the delta, dW_c and db_c;
  gradients every map's dW and db from the step's delta and the input the map read (part (c)'s check), with the
           intermediate term of dW_{N+1} and db_{N+1};
  padding  every delta's padded frames are +0.0.
  sweeps   at each clipped-ReLU temporal layer: For (and Back) as float64 steps from the step's own state of the step
           before (_steps and _bound of test_sweep_gpu.py), from the pre-activation the map wrote, recomputed at the
           step's plan where For + Back overwrote it, and X_i = For + Back bit for bit; dh, the delta the BPTT starts
           from (unstacked, with the D_aux term at interLayer), recomputed at the step's plans and checked; the BPTT from
           it, in place when uni-directional, else recomputed with ctcb_brnn_sweep_f32 and equal as dFor + dBack to the
           step's delta bit for bit;
  D_aux    against lambda times the float64 CTC gradient of the step's own A over the frames of layer m (bound of
           test_ctc_plans_gpu.py at the step's plan, plus one rounding for lambda).
  LSTM     the pre-activation recomputed at the step's plan and checked; the standalone sweep (plain, peephole or
           zoneout, U and P as the step read them, the layer's own lengths, zoneout's layer i, step and utterance
           numbering) from it on fresh buffers equals the step's gates, h and c bit for bit, which are checked against a
           float64 step from the step's own state (C_FWD, C_ACT of test_lstm_plans_gpu.py, with the lambdas); padded
           frames +0.0; the map above reads For + Back bit for bit; dh (+ D_aux W_{N+1}, or D'_m + dA W_{N+1} at the
           conditioned layer) recomputed and checked, the standalone BPTT from it equal to the step's dz bit for bit,
           and dz against net_oracle.lstm_direction_bptt (C_BPTT);
  recurrent every temporal layer's dU, or Wtf / Wtb, and dP (rec_grads of test_step_reductions_gpu.py), from the dz,
           dFor / dBack the call left or the BPTT recomputed (top-down where a uni-directional pair was reused).
Negative controls: the reference with a plausible wrong wiring (alpha omitted, the D_aux term dropped, X_m for X'_m,
the raw features, the clean parameters, gamma omitted, the dropout draw of the next step, the full-rate lengths at a
reduced layer m, the other direction's U, the clean U, P omitted, the zoneout draw of the next step or numbered by u,
direction 1 unshifted, dp_o from c_prev) must exceed the same bound at least 10 times on the same arrays.
Each net prints its ratios as one JSON line (pytest -s); the ledger test asserts which paths were reached."""
import ctypes
import json

import numpy as np
import pytest

from test_gemm_plans_gpu import BOUNDS as GEMM_BOUNDS, _chain as gemm_chain
from net_oracle import keep_mask
from test_ctc_plans_gpu import BOUNDS as CTC_BOUNDS, _plan as ctc_plan
from test_layernorm_gpu import C_FWD as C_LN, _fwd64 as ln_fwd64
from net_oracle import zoneout_masks
from test_lstm_plans_gpu import C_ACT, C_BPTT, C_FWD, _check_bptt, _check_forward
from test_sweep_gpu import MAXACT, _bound as sweep_bound, _plan as sweep_plan, _steps as sweep_steps
from test_step_reductions_gpu import (C_SOFTMAX, D_IN, MAXB, MAXT, NEG, NETS as MAP_NETS, U, _batches, _colsum_bound,
                                      _colsum_plan, _gemm_plan, _hook, _ratio, _rec_from_hooks, _softmax_check,
                                      _ws_array, peep_idx, rec_grads)

pytestmark = pytest.mark.gpu
STEP = 5                   # the step counter of every call: dropout, zoneout and weight noise draw from it
SHARD = (1, 2)             # the call's utterances are minibatch entries FIRST + STRIDE u (an emulated rank 1 of 2)
FIRST, STRIDE = SHARD
NETS = dict(MAP_NETS)
NETS.update({
    # the intermediate CTC at a ReLU layer with layer norm and dropout, and at a temporal layer
    "inter_relu_ln_dropout": dict(H=64, N=4, K=30, kw=dict(temporalLayer=3, layerNorm=True, dropout=0.1, interLayer=1,
                                                           interWeight=0.4)),
    "inter_temporal": dict(H=48, N=3, K=29, kw=dict(temporalLayer=2, interLayer=2, interWeight=0.5)),
    # subsampling below m: the intermediate CTC at the reduced rate
    "inter_sub_below": dict(H=64, N=4, K=30, kw=dict(temporalLayer=3, subsample=2, subsampleLayer=2, interLayer=2,
                                                     interWeight=0.3, dropout=0.1)),
    # self-conditioning below, at and above the temporal layers
    "cond_below": dict(H=64, N=3, K=30, kw=dict(temporalLayer=2, interLayer=1, interWeight=0.5, selfCondition=True)),
    "cond_at_lstm": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm", interLayer=2, interWeight=0.5,
                                                  selfCondition=True)),
    "cond_above_uni_dropout": dict(H=48, N=4, K=29, kw=dict(temporalLayer=1, unidirectional=True, interLayer=2,
                                                            interWeight=0.5, selfCondition=True, dropout=0.1)),
    "noise_ln": dict(H=64, N=3, K=31, kw=dict(temporalLayer=2, layerNorm=True, weightNoise=0.05)),
    "masks": dict(H=64, N=3, K=30, kw=dict(temporalLayer=2, freqMasks=2, freqMaskWidth=5, timeMasks=2,
                                           timeMaskWidth=6)),
    "zoneout_peep": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm", peephole=True, zoneoutCell=0.2,
                                                  zoneoutHidden=0.15)),
    # widths at which the forward and delta contractions run on the tensor cores; N ragged
    "dnn_h128_ln_dropout": dict(H=128, N=3, K=40, kw=dict(layerNorm=True, dropout=0.1)),
    "bi_h200_inter": dict(H=200, N=3, K=35, kw=dict(temporalLayer=2, interLayer=1, interWeight=0.3)),
    "uni_h256_cond_noise_masks": dict(H=256, N=3, K=37, kw=dict(temporalLayer=2, unidirectional=True, interLayer=1,
                                                                interWeight=0.3, selfCondition=True,
                                                                weightNoise=0.02, freqMasks=1, freqMaskWidth=4,
                                                                timeMasks=1, timeMaskWidth=4)),
    # the stacked map reads k H = 512 columns over about 140 rows: the tensor-core contraction splits over K
    "uni_h256_sub2_splitk": dict(H=256, N=3, K=33, kw=dict(temporalLayer=2, unidirectional=True, subsample=2,
                                                          subsampleLayer=2)),
    # the tensor-core ReLU sweep; the LSTM sweep with U in registers (KI = 32)
    "bi_relu_h1024": dict(H=1024, N=2, K=30, kw=dict(temporalLayer=1)),
    "lstm_uni_h1024": dict(H=1024, N=2, K=30, kw=dict(temporalLayer=1, cell="lstm", unidirectional=True)),
    # dh of an LSTM layer with the D_aux term; a dh pair used by layers j and j + 2; reduced lengths; the noisy U
    "lstm_inter": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm", interLayer=2, interWeight=0.4)),
    "lstm_uni_stack3_peep": dict(H=33, N=4, K=28, kw=dict(temporalLayer=1, numTemporal=3, cell="lstm",
                                                          unidirectional=True, peephole=True)),
    "lstm_sub_above": dict(H=32, N=4, K=28, kw=dict(temporalLayer=3, cell="lstm", subsample=2, subsampleLayer=2)),
    "lstm_noise_peep": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm", peephole=True, weightNoise=0.05)),
})
LEDGER = dict(kernels={}, splitk=set(), stages=set(), sweeps=set(), lstm_ki=set(), missing={}, rec={})
# the stage kinds every feature must reach somewhere in the table
WANT_STAGES = {
    "fwd_map", "fwd_logits", "fwd_stack", "ln_fwd", "ln_stats", "dropout", "delta", "delta_unstack", "ln_bwd",
    "inter_A", "inter_delta", "cond_A", "cond_P", "cond_X", "cond_Dm", "cond_dP", "cond_dA", "cond_delta", "cond_dWc",
    "cond_dbc", "head_dW", "head_db", "maps_dW", "maps_db", "masked_input", "noisy_params", "padding", "sweep_fwd",
    "bptt_dh", "bptt", "D_aux", "lstm_pre", "lstm_sweep", "lstm_bptt", "lstm_dh", "lstm_out", "rec_dW", "peep_dP",
    "cond_dh_lstm",
}


def _want(nn):
    """The stage kinds a net must reach, by its features."""
    w = {"fwd_map", "fwd_logits", "delta", "maps_dW", "maps_db", "padding"}
    if nn.numTemporal:
        w.add("rec_dW")
    if nn.numTemporal and nn.cell == "relu":
        w |= {"sweep_fwd", "bptt_dh"}
    if nn.numTemporal and nn.cell == "lstm":
        w |= {"lstm_pre", "lstm_sweep", "lstm_bptt"}
        if any(_temporal(nn, i) and i != _cond(nn) for i in range(1, nn.numLayers + 1)):
            w.add("lstm_dh")
        if nn.peephole:
            w.add("peep_dP")
        if nn.selfCondition and _temporal(nn, nn.interLayer):
            w.add("cond_dh_lstm")
    if nn.subsample > 1:
        w.add("fwd_stack")
    if nn.layerNorm:
        w |= {"ln_fwd", "ln_stats", "ln_bwd"}
    if nn.dropout:
        w.add("dropout")
    if nn.interLayer:
        w |= {"head_dW", "head_db", "D_aux"}
        w |= {"cond_A", "cond_P", "cond_X", "cond_Dm", "cond_dP", "cond_dA", "cond_dWc", "cond_dbc"} if nn.selfCondition \
            else {"inter_A", "inter_delta"}
    if nn.inputMasks:
        w.add("masked_input")
    if nn.weightNoise:
        w.add("noisy_params")
    return w


# ------------------------------------------------------------------------------------------------ helpers
def _net(c):
    import nnets.brnnet as brnnet
    import torch
    np.random.seed(17)
    nn = brnnet.NNet(D_IN, c["K"], c["H"], c["N"], MAXT, maxUtts=MAXB, maxLabels=6, **c["kw"])
    nn.initParams()
    rng = np.random.RandomState(2)        # biases off 0, so a padded frame's activations are not 0 on their own
    for w, b in nn.stack[:c["N"] + 1]:
        b.copy_(torch.from_numpy((0.1 * rng.randn(*b.shape)).astype(np.float32)))
    if nn.selfCondition:                  # W_c, b_c off 0, so X'_m differs from X_m
        nn.stack[-1][0].copy_(torch.from_numpy(rng.uniform(-0.4, 0.4, tuple(nn.stack[-1][0].shape)).astype(np.float32)))
        nn.stack[-1][1].copy_(torch.from_numpy(rng.uniform(-0.1, 0.1, tuple(nn.stack[-1][1].shape)).astype(np.float32)))
    for k in range(nn.peepholeEntries()):     # peepholes off 0, so an omitted P shows
        pk = nn.stack[len(nn.stack) - (1 if nn.selfCondition else 0) - nn.peepholeEntries() + k][0]
        pk.copy_(torch.from_numpy(rng.uniform(-0.5, 0.5, tuple(pk.shape)).astype(np.float32)))
    for i in nn.normedLayers():           # gamma off 1 and beta off 0, so a missing gamma or beta shows
        g, be = nn.stack[_ln_idx(nn, i)]
        g.copy_(torch.from_numpy((1.0 + 0.5 * rng.randn(*g.shape)).astype(np.float32)))
        be.copy_(torch.from_numpy((0.1 * rng.randn(*be.shape)).astype(np.float32)))
    if nn.dropoutStep is not None:
        nn.dropoutStep.fill_(STEP)
    return nn


def _temporal(nn, i):
    return nn.numTemporal and nn.temporalLayer <= i < nn.temporalLayer + nn.numTemporal


def _reduced(nn, i):
    return nn.subsample > 1 and i >= nn.subsampleLayer


def _normed(nn, i):
    return nn.layerNorm and 1 <= i <= nn.numLayers and not _temporal(nn, i)


def _cond(nn):
    return nn.interLayer if nn.selfCondition else 0


class Call:
    """The arrays of one training call: frames, lens and the device workspace views."""

    def __init__(self, nn, batch, lens, labels):
        self.nn, self.batch, self.B, self.lens, self.labels = nn, batch, batch.B, lens, labels
        self.grads = nn.grads.cpu().numpy()
        self.rdelta = {}           # map j: (device, host) of its delta, recomputed where the call overwrote it
        self.rec_done = set()      # the temporal layers whose recurrent gradients were checked

    def T(self, i):
        return self.nn.frames(self.batch.Tmax) if _reduced(self.nn, i) else self.batch.Tmax

    def R(self, i):
        return self.T(i) * self.B

    def Tu(self, i):
        return [self.nn.frames(t) if _reduced(self.nn, i) else t for t in self.lens]

    def ws(self, what, layer, T):
        """(device [T][B][width] view, host float32 [T*B][width]) of hook entry (what, layer)."""
        off, w = _hook(self.nn, what, layer)
        d = _ws_array(self.nn, off, T, self.B, w)
        return d, d.cpu().numpy().reshape(T * self.B, w)

    def tensor(self, idx, part, noisy=True):
        """(host float32 array, device pointer) of stack[idx][part] as the step read it: the noisy copy with noise on."""
        nn = self.nn
        v = nn.stack[idx][part]
        if noisy and nn.weightNoise > 0.0:
            off, n = _hook(nn, 19, 0)
            flat = nn._ws[off:off + 4 * n].view(nn._torch.float32)
            o = (v.data_ptr() - nn.params.data_ptr()) // 4
            d = flat[o:o + v.numel()].view(*v.shape)
            return d.cpu().numpy(), d.data_ptr()
        return v.cpu().numpy(), v.data_ptr()

    def act(self, i):
        """(host [R][width] float32, device pointer) of layer i's output as map i + 1 and the head read it."""
        nn, T = self.nn, self.T(i)
        if _temporal(nn, i) and nn.unidirectional:
            d, h = self.ws(1, i, T)
            return h, d.data_ptr()
        if _temporal(nn, i) and nn.cell == "lstm":      # Out = For + Back in float32 (the step's add2)
            df, f = self.ws(1, i, T)
            _, b = self.ws(2, i, T)
            return f + b, df.data_ptr()
        d, h = self.ws(0, i, T)
        return h, d.data_ptr()

    def map_input(self, j):
        """(host [R][cols], device pointer) of what map j read: the masked copy, S, X'_m or layer j - 1."""
        nn = self.nn
        if nn.subsample > 1 and j == nn.subsampleLayer:
            d, h = self.ws(6, 0, self.T(j))
            return h, d.data_ptr()
        if j == 1:
            if nn.inputMasks:
                d, h = self.ws(18, 0, self.T(1))
                return h, d.data_ptr()
            x = self.batch.d_feats[:self.R(1) * nn.inputDim]
            return x.cpu().numpy().reshape(self.R(1), nn.inputDim), x.data_ptr()
        if j - 1 == _cond(nn):
            d, h = self.ws(12, 0, self.T(j - 1))
            return h, d.data_ptr()
        return self.act(j - 1)


def _note(kind, plan, K):
    LEDGER["kernels"].setdefault(kind, set()).add(plan["kernel"])
    if plan["splits"] > 1:
        LEDGER["splitk"].add(kind)
    return (lambda c0, c1: c0 + c1 * gemm_chain(plan, K))(*GEMM_BOUNDS[plan["kernel"]])


def _plan(ta, tb, M, N, K, a, lda, b, ldb):
    from _ctcb import lib, check
    from test_gemm_plans_gpu import FIELDS
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan(ta, tb, M, N, K, a, lda, b, ldb, 1, out))
    return dict(zip(FIELDS, list(out)))


def _mm(A, B, alpha=1.0):
    """(alpha A B, |alpha| |A| |B|) in float64."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    return alpha * (A @ B), abs(alpha) * (np.abs(A) @ np.abs(B))


def _cmp(got, want, bound, relu=False, mask=None):
    """Ratio of float32 `got` to float64 `want` under `bound`; ReLU on want; masked entries (not mask > 0) must be
    exactly +0.0."""
    got = np.asarray(got)
    want = np.maximum(want, 0.0) if relu else want
    if mask is not None:
        off = ~(mask > 0)
        if got[off].view(np.uint32).any():
            return float("inf")
        return _ratio(np.where(off, 0.0, np.abs(got - want)), bound)
    return _ratio(np.abs(got - want), bound)


def _recompute(ta, tb, M, N, K, alpha, a, lda, b, ldb, beta=0.0, c0=None, mask=None, step_plan=None, bias=None,
               relu=False):
    """ctcb_gemm_f32 into fresh 256-byte-aligned scratch (C0 copied in when beta != 0), at the plan of the step's call."""
    import _ctcb
    import torch
    from _ctcb import lib, check
    out = torch.zeros(M * N, dtype=torch.float32, device="cuda")
    if c0 is not None:
        out.copy_(torch.from_numpy(np.ascontiguousarray(c0, np.float32).reshape(-1)).cuda())
    assert _plan(ta, tb, M, N, K, a, lda, b, ldb) == step_plan
    wsb = int(lib.ctcb_gemm_workspace_bytes(M, N, K))
    ws = torch.zeros(max(wsb, 16), dtype=torch.uint8, device="cuda")
    check(lib.ctcb_gemm_f32(ta, tb, M, N, K, alpha, a, lda, b, ldb, beta, out.data_ptr(), N, bias, int(relu),
                            None if mask is None else mask, ws.data_ptr(), wsb, _ctcb.current_stream()))
    torch.cuda.synchronize()
    return out, out.cpu().numpy().reshape(M, N)


def _ln_bwd(g, z, mu, rstd, gamma):
    """(dz64, bound) of the layer-norm backward from float32 g, z, Mu, Rstd, gamma (test_layernorm_gpu.py)."""
    g64, gam = g.astype(np.float64), gamma.astype(np.float64).reshape(1, -1)
    mu, rstd = mu.astype(np.float64).reshape(-1, 1), rstd.astype(np.float64).reshape(-1, 1)
    xh = (z.astype(np.float64) - mu) * rstd
    gh = g64 * gam
    a = gh.mean(axis=1, keepdims=True)
    b = (gh * xh).mean(axis=1, keepdims=True)
    bound = C_LN * U * rstd * (np.abs(gh) + np.abs(gh).mean(axis=1, keepdims=True) +
                               np.abs(xh) * (np.abs(gh * xh).mean(axis=1, keepdims=True) + np.abs(b)))
    return rstd * (gh - a - xh * b), bound


def _unstack(dS, T, B, n, k, Tu):
    """[T'][B][k n] -> [T][B][n] by frames t = k t' + j, 0 beyond each utterance's length."""
    Tp = dS.shape[0] // B
    d = dS.reshape(Tp, B, k, n).transpose(0, 2, 1, 3).reshape(Tp * k, B, n)[:T].copy()
    for u in range(B):
        d[Tu[u]:, u] = 0.0
    return d.reshape(T * B, n)


# ------------------------------------------------------------------------------------------------ sweeps and the CTC
def _keep(nn, i, c, step):
    """[T*B][H] keep mask of hidden layer i of the call's utterances (g = FIRST + STRIDE u) at `step`, as the device
    draws it."""
    T, H = c.T(i), nn.layerSize
    k = np.stack([keep_mask(nn.dropout, nn.dropoutSeed, step, i, FIRST + STRIDE * u, T, H) for u in range(c.B)],
                 axis=1)
    return k.reshape(T * c.B, H)


def _noisy_ptr(c, idx, part):
    return c.tensor(idx, part)[1]


def _rec(c, i):
    """[(host W, device pointer)] of temporal layer i's recurrent matrices, one per direction."""
    nn = c.nn
    ndir = 1 if nn.unidirectional else 2
    base = nn.numLayers + 1 + (i - nn.temporalLayer) * ndir
    return [c.tensor(base + d, 0) for d in range(ndir)]


class _Sw:
    def __init__(self, T, lens, ndir):
        self.T, self.lens, self.ndir = T, np.asarray(lens), ndir


def _sweep_ratio(c, i, outs, inputs, Ms, acts):
    nn = c.nn
    ndir = len(Ms)
    plan = sweep_plan(nn.layerSize, c.B, ndir)
    LEDGER["sweeps"].add(plan["kernel"])
    C = sweep_bound(plan, nn.layerSize)
    T, H = c.T(i), nn.layerSize
    r = lambda a: np.asarray(a, np.float32).reshape(T, c.B, H)       # noqa: E731
    w = sweep_steps(_Sw(T, c.Tu(i), ndir), [r(o) for o in outs], r(inputs), Ms,
                    None if acts is None else [r(a) for a in acts], C)
    return w["ratio"] / C


def _relu_sweep_fwd(c, i, pre, rep):
    """For (and Back) of ReLU temporal layer i: float64 steps from the step's own states of the step before, from the
    pre-activation the map wrote (recomputed where For + Back overwrote it); X_i = For + Back in float32, bit for bit."""
    nn = c.nn
    T = c.T(i)
    W = _rec(c, i)
    outs = [c.ws(1, i, T)[1]] + ([] if nn.unidirectional else [c.ws(2, i, T)[1]])
    rep["sweep_fwd%d" % i] = _sweep_ratio(c, i, outs, pre, [w.T for w, _ in W], None)
    if not nn.unidirectional:
        X = c.ws(0, i, T)[1]
        assert np.array_equal(X.view(np.uint32), (outs[0] + outs[1]).view(np.uint32)), "X_%d != For + Back" % i
    LEDGER["stages"].add("sweep_fwd")


def _dh(c, i, rep, neg):
    """(device dh, host dh [R][H]) of temporal layer i: delta_{i+1} W_{i+1} (the step's delta of map i + 1, or the one
    recomputed above where the call overwrote it), unstacked below map L, + D_aux W_{N+1} at interLayer, recomputed at
    the step's plans and checked; None where the delta of map i + 1 is not known."""
    import torch
    nn = c.nn
    N, B, H, K = nn.numLayers, c.B, nn.layerSize, nn.outputDim
    T, R = c.T(i), c.R(i)
    if _hook(nn, 7, i + 1) is not None:
        dd, d = c.ws(7, i + 1, c.T(i + 1))
    elif i + 1 in c.rdelta:
        dd, d = c.rdelta[i + 1]
    else:
        return None
    n_out = d.shape[1]
    W, Wp = c.tensor(i, 0)
    n_in = W.shape[1]
    R1 = c.R(i + 1)
    plan = _plan(0, 0, R1, n_in, n_out, dd.data_ptr(), n_out, Wp, n_in)
    cb = _note("delta", plan, n_out)
    dh_d, dh = _recompute(0, 0, R1, n_in, n_out, 1.0, dd.data_ptr(), n_out, Wp, n_in, step_plan=plan)
    P, S = _mm(d, W)
    bound = cb * U * S
    if nn.subsample > 1 and i + 1 == nn.subsampleLayer:
        dh, P, bound = (_unstack(a, T, B, H, nn.subsample, c.Tu(i)) for a in (dh, P, bound))
        dh_d = torch.from_numpy(np.ascontiguousarray(dh, np.float32).reshape(-1)).cuda()
        LEDGER["stages"].add("delta_unstack")
    if i == nn.interLayer:
        Dd, Da = c.ws(9, 0, T)
        Wo, Wop = c.tensor(N, 0)
        plan2 = _plan(0, 0, R, H, K, Dd.data_ptr(), K, Wop, H)
        cb2 = _note("inter_delta", plan2, K)
        dh_d, dh2 = _recompute(0, 0, R, H, K, 1.0, Dd.data_ptr(), K, Wop, H, beta=1.0, c0=dh, step_plan=plan2)
        P2, S2 = _mm(Da, Wo)
        bound = bound + cb2 * U * (S2 + np.abs(P))
        neg.setdefault("D_aux_dropped", []).append(_ratio(np.abs(dh2 - P), bound))
        P, dh = P + P2, dh2
        LEDGER["stages"].add("inter_delta")
    kind = "lstm_dh" if nn.cell == "lstm" else "bptt_dh"
    rep["%s%d" % (kind, i)] = _ratio(np.abs(dh - P), bound)
    LEDGER["stages"].add(kind)
    return dh_d, dh


def _relu_bptt(c, i, rep, neg):
    """The BPTT of ReLU temporal layer i from its dh (_dh): the uni-directional result in place where the call left it,
    else recomputed with ctcb_brnn_sweep_f32 (and then the delta of map i for the layer below); the bi-directional one
    recomputed and equal, as For + Back, to the step's delta bit for bit.  Then the recurrent gradients from it."""
    import _ctcb
    import torch
    from _ctcb import lib, check
    nn = c.nn
    B, H = c.B, nn.layerSize
    T, R = c.T(i), c.R(i)
    got = _dh(c, i, rep, neg)
    if got is None:
        return
    dh_d, dh = got
    Wr = _rec(c, i)
    acts = [c.ws(1, i, T)[1]] + ([] if nn.unidirectional else [c.ws(2, i, T)[1]])
    if nn.unidirectional and _hook(nn, 7, i) is not None:
        dd = c.ws(7, i, T)
        dF, ptrs = [dd[1]], (dd[0].data_ptr() + 4 * B * H, None, c.ws(1, i, T)[0].data_ptr(), None, H)
    else:
        outs = [torch.zeros(R * H, dtype=torch.float32, device="cuda") for _ in range(len(Wr))]
        lens_d = torch.tensor(c.Tu(i), dtype=torch.int32, device="cuda")
        wsb = int(lib.ctcb_brnn_sweep_workspace_bytes(H, B))
        scr = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        bi = not nn.unidirectional
        check(lib.ctcb_brnn_sweep_f32(1, T, B, H, lens_d.data_ptr(), dh_d.data_ptr(), Wr[0][1],
                                      Wr[1][1] if bi else None, outs[0].data_ptr(), outs[1].data_ptr() if bi else None,
                                      c.ws(1, i, T)[0].data_ptr(), c.ws(2, i, T)[0].data_ptr() if bi else None,
                                      MAXACT, scr.data_ptr(), wsb, _ctcb.current_stream()))
        torch.cuda.synchronize()
        dF = [o.cpu().numpy().reshape(R, H) for o in outs]
        if bi:
            got = c.ws(7, i, T)[1]
            assert np.array_equal(got.view(np.uint32), (dF[0] + dF[1]).view(np.uint32)), \
                "the delta of map %d is not the BPTT of its recomputed dh" % i
            ptrs = (outs[0].data_ptr() + 4 * B * H, outs[1].data_ptr(), c.ws(1, i, T)[0].data_ptr(),
                    c.ws(2, i, T)[0].data_ptr() + 4 * B * H, H)
        else:                                    # a later layer of the stack wrote the pair: the delta of map i
            c.rdelta[i] = (outs[0], dF[0])
            ptrs = (outs[0].data_ptr() + 4 * B * H, None, c.ws(1, i, T)[0].data_ptr(), None, H)
    rep["bptt%d" % i] = _sweep_ratio(c, i, dF, dh, [w for w, _ in Wr], acts)
    LEDGER["stages"].add("bptt")
    r = lambda a: np.asarray(a).reshape(T, B, H)      # noqa: E731
    _rec_check(c, i, rec_grads(nn, i - nn.temporalLayer, T, c.Tu(i), [r(x) for x in dF], [r(a) for a in acts], None,
                               ptrs, c.grads, None, neg), rep)


def _rec_check(c, i, out, rep):
    rep["rec%d" % i] = {k: v for k, v in out.items() if not k.startswith("kernel")}
    LEDGER["stages"].add("rec_dW")
    if any(k.startswith("dP") for k in out):
        LEDGER["stages"].add("peep_dP")
    c.rec_done.add(i)


# ------------------------------------------------------------------------------------------------ LSTM layers
def _lstm_sweep(c, i, mode, gates, hs, cs, dh=None, dz=None):
    """ctcb_lstm_sweep_f32 / _peephole_f32 / _zoneout_f32, as the net calls for, on device buffers: mode 0 the forward
    from pre-activations in `gates`, mode 1 the BPTT from dh into dz; U and P as the step read them."""
    import _ctcb
    import torch
    from _ctcb import lib, check
    nn = c.nn
    T, B, H = c.T(i), c.B, nn.layerSize
    j = i - nn.temporalLayer
    nd = len(hs)
    Us = [p for _, p in _rec(c, i)]
    Ps = [c.tensor(peep_idx(nn, j, d), 0)[1] for d in range(nd)] if nn.peephole else [None, None]
    lens = torch.tensor(c.Tu(i), dtype=torch.int32, device="cuda")
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    two = lambda xs: (p(xs[0]), p(xs[1]) if nd == 2 else None)     # noqa: E731
    Uf, Ub = Us[0], Us[1] if nd == 2 else None
    Pf, Pb = Ps[0], Ps[1] if nd == 2 else None
    hF, hB = two(hs) if mode == 0 else (None, None)
    cF, cB = two(cs)
    st = _ctcb.current_stream()
    if nn.zoneout:
        n = int(lib.ctcb_lstm_sweep_zoneout_workspace_bytes(H, B))
        ws = torch.zeros(n, dtype=torch.uint8, device="cuda")
        rc = lib.ctcb_lstm_sweep_zoneout_f32(mode, T, B, H, p(lens), p(gates), Uf, Ub, Pf, Pb, hF, hB, cF, cB, p(dh),
                                             p(dz), nn.zoneoutCell, nn.zoneoutHidden, 1,
                                             nn.dropoutSeed & 0xFFFFFFFFFFFFFFFF, p(nn.dropoutStep), FIRST, STRIDE, i,
                                             p(ws), n, st)
    else:
        n = int(lib.ctcb_lstm_sweep_workspace_bytes(H, B))
        ws = torch.zeros(n, dtype=torch.uint8, device="cuda")
        if nn.peephole:
            rc = lib.ctcb_lstm_sweep_peephole_f32(mode, T, B, H, p(lens), p(gates), Uf, Ub, Pf, Pb, hF, hB, cF, cB,
                                                  p(dh), p(dz), p(ws), n, st)
        else:
            rc = lib.ctcb_lstm_sweep_f32(mode, T, B, H, p(lens), p(gates), Uf, Ub, hF, hB, cF, cB, p(dh), p(dz), p(ws),
                                         n, st)
    check(rc)
    torch.cuda.synchronize()
    assert int(ws[:4].view(torch.int32).item()) == 0, "the LSTM sweep set its error flag"


class _Prob:
    """What _check_forward / _check_bptt of test_lstm_plans_gpu.py read of a sweep problem."""

    def __init__(self, c, i, pre, Us, Ps, dh=None):
        nn = c.nn
        self.H, self.T, self.B = nn.layerSize, c.T(i), c.B
        self.ndir = len(Us)
        self.lens = np.asarray(c.Tu(i))
        self.pre = pre.reshape(self.T, self.B, -1)
        self.Us, self.Ps = Us, Ps
        self.dh = None if dh is None else dh.reshape(self.T, self.B, self.H)


def _lambdas(c, i, step=STEP, numbered=None):
    """Per direction [T][B][H] lambda_c, lambda_h of layer i as the device draws them (None without zoneout); numbered:
    the minibatch index of utterance u (FIRST + STRIDE u by default)."""
    nn = c.nn
    if not nn.zoneout:
        return None, None
    T, H = c.T(i), nn.layerSize
    g = numbered or (lambda u: FIRST + STRIDE * u)
    nd = 1 if nn.unidirectional else 2
    m = [[zoneout_masks(nn.zoneoutCell, nn.zoneoutHidden, nn.dropoutSeed, step, i, d, g(u), T, H) for u in range(c.B)]
         for d in range(nd)]
    return ([np.stack([x[0] for x in md], axis=1).astype(np.float64) for md in m],
            [np.stack([x[1] for x in md], axis=1).astype(np.float64) for md in m])


def _lstm_state(c, i):
    """The step's gates (device, host [T][B][G]), h and c per direction (device, host [T][B][H])."""
    nn = c.nn
    T, B, H = c.T(i), c.B, nn.layerSize
    nd = 1 if nn.unidirectional else 2
    g = c.ws(3, i, T)
    hs = [c.ws(1 + d, i, T) for d in range(nd)]
    cs = [c.ws(4 + d, i, T) for d in range(nd)]
    sh = lambda x: x[1].reshape(T, B, -1)      # noqa: E731
    return g, [sh(x) for x in hs], [sh(x) for x in cs], hs, cs, sh(g)


def _lstm_forward(c, i, pre_d, pre, rep, neg):
    """LSTM layer i from the pre-activation the map wrote (recomputed, as the gates overwrote it): the forward sweep on
    fresh buffers equals the step's gates, h and c bit for bit; those against a float64 step from the step's own state
    of the step before (C_FWD, C_ACT), with zoneout's lambdas and kept values; padded frames +0.0."""
    import torch
    nn = c.nn
    T, B, H = c.T(i), c.B, nn.layerSize
    nd = 1 if nn.unidirectional else 2
    j = i - nn.temporalLayer
    plan = (ctypes.c_int32 * 4)()
    from _ctcb import lib
    debug = lib.ctcb_debug_lstm_zoneout_plan if nn.zoneout else lib.ctcb_debug_lstm_plan
    assert debug(H, B, nd, int(nn.peephole), plan) == 0
    LEDGER["lstm_ki"].add(int(plan[0]))
    gates = pre_d.clone()
    hs = [torch.zeros(T * B * H, dtype=torch.float32, device="cuda") for _ in range(nd)]
    cs = [torch.zeros(T * B * H, dtype=torch.float32, device="cuda") for _ in range(nd)]
    _lstm_sweep(c, i, 0, gates, hs, cs)
    _, sh, sc, _, _, sg = _lstm_state(c, i)
    for name, a, b in [("gates", gates, sg)] + [("h%d" % d, hs[d], sh[d]) for d in range(nd)] + \
            [("c%d" % d, cs[d], sc[d]) for d in range(nd)]:
        assert np.array_equal(a.cpu().numpy().view(np.uint32), b.reshape(-1).view(np.uint32)), \
            "layer %d: the sweep of the recomputed pre-activation gives other %s than the step" % (i, name)
    for u, t in enumerate(c.Tu(i)):
        assert not any(x[t:, u].view(np.uint32).any() for x in [sg] + sh + sc), "a padded frame of layer %d" % i
    LEDGER["stages"].add("lstm_sweep")
    U_ = [w for w, _ in _rec(c, i)]
    P_ = [c.tensor(peep_idx(nn, j, d), 0)[0] for d in range(nd)] if nn.peephole else None
    r = dict(gates=sg, h=sh, c=sc)
    lc, lh = _lambdas(c, i)
    f = _check_forward(r, _Prob(c, i, pre, U_, P_), lc, lh)
    rep["lstm_fwd%d" % i] = dict(gates=f["gates"] / C_FWD, c=f["c"] / C_FWD, h=f["h"] / C_FWD,
                                 act=f["act_exact"] / C_ACT)
    if lc is not None:
        assert f["kept"], "layer %d: a kept c or h does not carry the previous value's bytes" % i
    worst = lambda g: max(g["gates"], g["c"], g["h"]) / C_FWD      # noqa: E731
    if nd == 2:
        neg.setdefault("other_direction_U", []).append(
            _check_forward(r, _Prob(c, i, pre, U_[::-1], P_), lc, lh)["gates"] / C_FWD)
    if nn.weightNoise > 0.0:
        clean = [c.tensor(nn.numLayers + 1 + j * nd + d, 0, noisy=False)[0] for d in range(nd)]
        neg.setdefault("clean_U", []).append(_check_forward(r, _Prob(c, i, pre, clean, P_), lc, lh)["gates"] / C_FWD)
    if nn.peephole:
        neg.setdefault("P_omitted", []).append(_check_forward(r, _Prob(c, i, pre, U_, None), lc, lh)["gates"] / C_FWD)
    if lc is not None:
        neg.setdefault("zoneout_draw_of_next_step", []).append(
            worst(_check_forward(r, _Prob(c, i, pre, U_, P_), *_lambdas(c, i, STEP + 1))))
        neg.setdefault("zoneout_numbered_by_u", []).append(
            worst(_check_forward(r, _Prob(c, i, pre, U_, P_), *_lambdas(c, i, numbered=lambda u: u))))


def _lstm_bptt(c, i, dh_d, dh, rep, neg):
    """The BPTT of LSTM layer i from its dh: the standalone sweep (mode 1) from the step's gates and c gives the step's
    dz (the delta of map i) bit for bit; dz against net_oracle.lstm_direction_bptt of the step's own activations
    (C_BPTT, the lambdas included); then the recurrent and peephole gradients from it."""
    import torch
    nn = c.nn
    T, B, H = c.T(i), c.B, nn.layerSize
    nd = 1 if nn.unidirectional else 2
    j = i - nn.temporalLayer
    g, sh, sc, hd, cd, sg = _lstm_state(c, i)
    dz = torch.zeros(T * B * nd * 4 * H, dtype=torch.float32, device="cuda")
    _lstm_sweep(c, i, 1, g[0].clone(), [None] * nd, [x[0].clone() for x in cd], dh=dh_d, dz=dz)
    got = c.ws(7, i, T)[1]
    assert np.array_equal(dz.cpu().numpy().view(np.uint32), got.reshape(-1).view(np.uint32)), \
        "the delta of map %d is not the LSTM BPTT of its recomputed dh" % i
    U_ = [w for w, _ in _rec(c, i)]
    P_ = [c.tensor(peep_idx(nn, j, d), 0)[0] for d in range(nd)] if nn.peephole else None
    r = dict(gates=sg, h=sh, c=sc, dz=got.reshape(T, B, -1))
    lc, lh = _lambdas(c, i)
    rep["lstm_bptt%d" % i] = _check_bptt(r, _Prob(c, i, sg, U_, P_, dh), lc, lh) / C_BPTT
    LEDGER["stages"].add("lstm_bptt")
    _rec_check(c, i, _rec_from_hooks(nn, c.batch, c.lens, j, c.grads, None, neg), rep)


def _daux(c, rep, neg):
    """D_aux against lambda times the float64 CTC gradient of the step's own A over T'_u frames at a reduced m (bound of
    test_ctc_plans_gpu.py at the step's plan, plus one rounding for lambda); padded frames exactly 0.  Negative
    control: the same reference over the full-rate lengths."""
    from oracle import ctc_oracle
    nn = c.nn
    m, K, B = nn.interLayer, nn.outputDim, c.B
    T = c.T(m)
    Ad, A = c.ws(8, 0, T)
    Dd, D = c.ws(9, 0, T)
    A, D = A.reshape(T, B, K), D.reshape(T, B, K)
    rc, plan = ctc_plan(B, T, K, nn.maxLabels, Ad.data_ptr(), Dd.data_ptr(), us=K, fs=B * K)
    assert rc == 0
    gb = CTC_BOUNDS[plan["kernel"]][0]
    lam = float(np.float32(nn.interWeight))

    def ref(u, t):
        x = A[:t, u].astype(np.float64)
        p = np.exp(x - x.max(axis=1, keepdims=True))
        p /= p.sum(axis=1, keepdims=True)
        _, g, skip = ctc_oracle.ctc_loss(np.asfortranarray(p.T), np.asarray(c.labels[u], np.int32))
        out = np.zeros((T, K))
        if not skip:
            out[:t] = lam * g.T
        return out

    r, wrong = 0.0, 0.0
    for u, t in enumerate(c.Tu(m)):
        assert not D[t:, u].view(np.uint32).any(), "a padded frame of D_aux is not +0.0"
        want = ref(u, t)
        bound = lam * gb + U * np.abs(want)
        r = max(r, _ratio(np.abs(D[:, u] - want), bound))
        if _reduced(nn, m) and min(c.lens[u], T) != t:
            wrong = max(wrong, _ratio(np.abs(D[:, u] - ref(u, min(c.lens[u], T))), bound))
    rep["D_aux"] = r
    if _reduced(nn, m):
        neg.setdefault("full_rate_lens", []).append(wrong)
    LEDGER["stages"].add("D_aux")


# ------------------------------------------------------------------------------------------------ the stages
def _forward(c, rep, neg):
    nn = c.nn
    N, B = nn.numLayers, c.B
    s = np.float32(1.0 / (1.0 - nn.dropout)) if nn.dropout > 0.0 else np.float32(1.0)
    for i in range(1, N + 2):
        R = c.R(i)
        n_out = nn._map_rows(i)
        x, xp = c.map_input(i)
        n_in = x.shape[1]
        if nn.subsample > 1 and i == nn.subsampleLayer:          # S: layer L - 1 stacked k frames at a time, exactly
            prev = (c.map_input(1)[0] if i == 1 else
                    (c.ws(12, 0, c.T(i - 1))[1] if i - 1 == _cond(nn) else c.act(i - 1)[0]))
            k, n = nn.subsample, prev.shape[1]
            T0, Tp = c.T(i - 1), c.T(i)
            want = np.zeros((Tp * k, B, n), np.float32)
            want[:T0] = prev.reshape(T0, B, n)
            for u in range(B):
                want[c.lens[u]:, u] = 0.0
            want = want.reshape(Tp, k, B, n).transpose(0, 2, 1, 3).reshape(Tp * B, k * n)
            assert np.array_equal(x.view(np.uint32), want.view(np.uint32)), "S is not the stack of layer %d" % (i - 1)
            LEDGER["stages"].add("fwd_stack")
        W, Wp = c.tensor(i - 1, 0)
        b, _ = c.tensor(i - 1, 1)
        plan = _plan(0, 1, R, n_out, n_in, xp, n_in, Wp, n_in)
        cb = _note("fwd", plan, n_in)
        P, S = _mm(x, W.T)
        P, S = P + b.reshape(1, -1), S + np.abs(b).reshape(1, -1)
        bound = cb * U * S
        relu = i <= N and not _temporal(nn, i)
        Pf = None
        if i == 1 and nn.inputMasks:                 # the raw features, where the masks changed them
            f = c.batch.d_feats[:R * nn.inputDim].cpu().numpy().reshape(R, nn.inputDim)
            if not np.array_equal(f, x):
                Pf = np.asarray(f, np.float64) @ W.T.astype(np.float64) + b.reshape(1, -1)
        if nn.weightNoise > 0.0:
            Wc_, _ = c.tensor(i - 1, 0, noisy=False)
            Pc = np.asarray(x, np.float64) @ Wc_.T.astype(np.float64) + b.reshape(1, -1)
        if _normed(nn, i):
            _, z = c.ws(15, i, c.T(i))
            _, mu = c.ws(16, i, c.T(i))
            _, rstd = c.ws(17, i, c.T(i))
            rep["fwd_z%d" % i] = r = _cmp(z, P, bound)
            LEDGER["stages"].add("fwd_map")
            g_, _ = c.tensor(_ln_idx(nn, i), 0)
            be, _ = c.tensor(_ln_idx(nn, i), 1)
            mu64, rstd64, y64, Xm = ln_fwd64(z, g_.reshape(1, -1).astype(np.float64), be.reshape(1, -1).astype(np.float64))
            M = np.abs(z.astype(np.float64)).mean(axis=1, keepdims=True)
            rep["ln_mu%d" % i] = _ratio(np.abs(mu.astype(np.float64) - mu64), C_LN * U * M)
            rep["ln_rstd%d" % i] = _ratio(np.abs(rstd.astype(np.float64) - rstd64),
                                          C_LN * U * rstd64 * (1.0 + C_LN * U * (M * rstd64) ** 2))
            LEDGER["stages"].update(("ln_fwd", "ln_stats"))
            y, ybound = y64, C_LN * U * (np.abs(g_.reshape(1, -1)) * Xm + np.abs(be.reshape(1, -1)))
            got_z, want_z = z, P
        else:
            y, ybound = (np.maximum(P, 0.0) if relu else P), bound
            got_z = None
        if _temporal(nn, i) and nn.cell == "relu":
            if nn.unidirectional:
                _, pre = c.ws(0, i, c.T(i))
            else:                                     # For + Back overwrote the pre-activation: recompute it
                _, pre = _recompute(0, 1, R, n_out, n_in, 1.0, xp, n_in, Wp, n_in, step_plan=plan,
                                    bias=nn.stack[i - 1][1].data_ptr() if nn.weightNoise == 0.0 else
                                    _noisy_ptr(c, i - 1, 1))
            rep["fwd_map%d" % i] = _cmp(pre, P, bound)
            LEDGER["stages"].add("fwd_map")
            _relu_sweep_fwd(c, i, pre, rep)
            continue
        if _temporal(nn, i):                          # the gates overwrote the pre-activation: recompute it
            pre_d, pre = _recompute(0, 1, R, n_out, n_in, 1.0, xp, n_in, Wp, n_in, step_plan=plan,
                                    bias=nn.stack[i - 1][1].data_ptr() if nn.weightNoise == 0.0 else
                                    _noisy_ptr(c, i - 1, 1))
            rep["fwd_map%d" % i] = _cmp(pre, P, bound)
            LEDGER["stages"].update(("fwd_map", "lstm_pre"))
            _lstm_forward(c, i, pre_d, pre, rep, neg)
            continue
        _, X = c.ws(0, i, c.T(i))
        below = i - 1
        if _temporal(nn, below) and nn.cell == "lstm" and not nn.unidirectional and below != _cond(nn) and \
                not (nn.subsample > 1 and i == nn.subsampleLayer) and not (nn.dropout > 0.0 and relu):
            # map i read Out = For + Back: the same contraction of For + Back in float32 gives its bytes
            import torch
            out_d = torch.from_numpy(np.ascontiguousarray(x, np.float32).reshape(-1)).cuda()
            _, again = _recompute(0, 1, R, n_out, n_in, 1.0, out_d.data_ptr(), n_in, Wp, n_in, step_plan=plan,
                                  bias=nn.stack[i - 1][1].data_ptr() if nn.weightNoise == 0.0 else
                                  _noisy_ptr(c, i - 1, 1), relu=relu and not _normed(nn, i))
            mine = c.ws(15, i, c.T(i))[1] if _normed(nn, i) else X
            assert np.array_equal(again.view(np.uint32), mine.view(np.uint32)), \
                "map %d did not read For + Back of LSTM layer %d" % (i, below)
            LEDGER["stages"].add("lstm_out")
        if nn.dropout > 0.0 and relu:
            keep = _keep(nn, i, c, STEP)
            assert not X[~keep].view(np.uint32).any(), "layer %d: a dropped entry is not +0.0" % i
            db = s * ybound + U * s * np.abs(y)
            r = _ratio(np.where(keep, np.abs(X - s * y), 0.0), db)
            rep["dropout%d" % i] = dict(ratio=r, dropped=int((~keep).sum()), kept=int(keep.sum()))
            assert (~keep).any(), "dropout on layer %d dropped nothing" % i
            neg.setdefault("alpha_fwd", []).append(_ratio(np.where(keep, np.abs(X - y), 0.0), db))
            neg.setdefault("dropout_draw_of_next_step", []).append(
                _ratio(np.abs(X - s * y * _keep(nn, i, c, STEP + 1)), db))
            LEDGER["stages"].add("dropout")
            rep["fwd_map%d" % i] = r
        elif got_z is None:
            rep["fwd_map%d" % i] = _cmp(X, P, bound, relu=relu)
        else:
            rep["ln_y%d" % i] = _ratio(np.abs(X - y), ybound)
        LEDGER["stages"].add("fwd_logits" if i == N + 1 else "fwd_map")
        out = got_z if got_z is not None else X
        if Pf is not None and not (nn.dropout and relu):
            neg.setdefault("raw_feats", []).append(_cmp(out, Pf, bound, relu=relu and got_z is None))
            LEDGER["stages"].add("masked_input")
        if nn.weightNoise > 0.0 and (got_z is not None or not (nn.dropout and relu)):
            neg.setdefault("clean_params", []).append(_cmp(out, Pc, bound, relu=relu and got_z is None))
            LEDGER["stages"].add("noisy_params")
        if i - 1 == _cond(nn) and i - 1 >= 1:         # map m + 1 must read X'_m, not X_m
            xm, _ = c.act(i - 1)
            Pm = np.asarray(xm, np.float64) @ W.T.astype(np.float64) + b.reshape(1, -1)
            if not (nn.dropout and relu):
                neg.setdefault("X_m_for_Xc", []).append(_ratio(np.abs(out - (np.maximum(Pm, 0) if relu and got_z is None
                                                                             else Pm)), bound))
    if nn.interLayer:
        _inter_forward(c, rep)


def _ln_idx(nn, i):
    """Index into nn.stack of [gamma, beta] of normalised layer i."""
    return len(nn.stack) - (1 if nn.selfCondition else 0) - nn.peepholeEntries() - len(nn.normedLayers()) + \
        nn.normedLayers().index(i)


def _inter_forward(c, rep):
    """A = X_m W_{N+1}^T + b_{N+1}; self-conditioned: P = softmax(A) and X'_m = X_m + P W_c^T + b_c."""
    nn = c.nn
    m, N, K, H, T = nn.interLayer, nn.numLayers, nn.outputDim, nn.layerSize, c.T(nn.interLayer)
    R = c.R(m)
    xm, xp = c.act(m)
    W, Wp = c.tensor(N, 0)
    b, _ = c.tensor(N, 1)
    _, A = c.ws(8, 0, T)
    plan = _plan(0, 1, R, K, H, xp, H, Wp, H)
    kind = "cond" if nn.selfCondition else "head"
    cb = _note(kind, plan, H)
    P, S = _mm(xm, W.T)
    rep["inter_A"] = _cmp(A, P + b.reshape(1, -1), cb * U * (S + np.abs(b).reshape(1, -1)))
    LEDGER["stages"].add("cond_A" if nn.selfCondition else "inter_A")
    if not nn.selfCondition:
        return
    dP, Pm = c.ws(13, 0, T)
    rep["cond_P"], _ = _softmax_check(A, Pm)
    Wc, Wcp = c.tensor(len(nn.stack) - 1, 0)
    bc, _ = c.tensor(len(nn.stack) - 1, 1)
    _, Xc = c.ws(12, 0, T)
    plan = _plan(0, 1, R, H, K, dP.data_ptr(), K, Wcp, K)
    cb = _note("cond", plan, K)
    P2, S2 = _mm(Pm, Wc.T)
    want = P2 + xm + bc.reshape(1, -1)
    rep["cond_X"] = _cmp(Xc, want, cb * U * (S2 + np.abs(xm) + np.abs(bc).reshape(1, -1)))
    LEDGER["stages"].update(("cond_P", "cond_X"))


def _backward(c, rep, neg):
    nn = c.nn
    N, B, H, K = nn.numLayers, c.B, nn.layerSize, nn.outputDim
    s = np.float32(1.0 / (1.0 - nn.dropout)) if nn.dropout > 0.0 else np.float32(1.0)
    for j in range(1, N + 2):                    # padded frames of every delta are +0.0
        h = _hook(nn, 7, j)
        if h is None:
            continue
        _, d = c.ws(7, j, c.T(j))
        d = d.reshape(c.T(j), B, -1)
        for u, t in enumerate(c.Tu(j)):
            assert not d[t:, u].view(np.uint32).any(), "map %d: a padded frame of the delta is not +0.0" % j
        LEDGER["stages"].add("padding")
    for i in range(N, 0, -1):
        if _temporal(nn, i) and i != _cond(nn):
            if nn.cell == "relu":
                _relu_bptt(c, i, rep, neg)
            else:
                got = _dh(c, i, rep, neg)
                if got is not None:
                    _lstm_bptt(c, i, *got, rep, neg)
            continue
        hd = _hook(nn, 7, i + 1)
        if hd is None:
            continue
        dd, d = c.ws(7, i + 1, c.T(i + 1))
        n_out = d.shape[1]
        W, Wp = c.tensor(i, 0)
        n_in = W.shape[1]
        n = H
        alpha = float(s) if nn.dropout > 0.0 else 1.0
        stacked = nn.subsample > 1 and i + 1 == nn.subsampleLayer
        cond = i == _cond(nn)
        if cond:
            _cond_backward(c, rep, neg, i, dd, d, W, Wp, alpha)
            continue
        maskh, maskp = (c.ws(6, 0, c.T(i + 1))[1], c.ws(6, 0, c.T(i + 1))[0].data_ptr()) if stacked else c.act(i)
        R1 = c.R(i + 1)
        plan = _plan(0, 0, R1, n_in, n_out, dd.data_ptr(), n_out, Wp, n_in)
        cb = _note("delta", plan, n_out)
        P, S = _mm(d, W, alpha)
        P1, S1 = _mm(d, W, 1.0)
        bound = cb * U * S
        mask = maskh
        if stacked:
            Tu = c.Tu(i)
            P = _unstack(P * (mask > 0), c.T(i), B, n, nn.subsample, Tu)
            P1 = _unstack(P1 * (mask > 0), c.T(i), B, n, nn.subsample, Tu)
            bound = _unstack(bound, c.T(i), B, n, nn.subsample, Tu)
            mask = _unstack(mask, c.T(i), B, n, nn.subsample, Tu)
            LEDGER["stages"].add("delta_unstack")
        inter = i == nn.interLayer
        if inter:
            Da = c.ws(9, 0, c.T(i))
            Wo, Wop = c.tensor(N, 0)
            plan2 = _plan(0, 0, c.R(i), n, K, Da[0].data_ptr(), K, Wop, n)
            cb2 = _note("inter_delta", plan2, K)
            P2, S2 = _mm(Da[1], Wo, alpha)
            noD = P
            P = P + P2
            bound = bound + cb2 * U * (S2 + np.abs(noD))
            LEDGER["stages"].add("inter_delta")
        if _normed(nn, i):                          # g was overwritten by dz: recompute it at the step's plan
            g_dev, g = _recompute(0, 0, R1, n_in, n_out, alpha, dd.data_ptr(), n_out, Wp, n_in, mask=maskp,
                                  step_plan=plan)
            if stacked:
                g = _unstack(g, c.T(i), B, n, nn.subsample, c.Tu(i))
            if inter:
                _, g = _recompute(0, 0, c.R(i), n, K, alpha, Da[0].data_ptr(), K, Wop, n, beta=1.0, c0=g,
                                  mask=maskp, step_plan=plan2)
            rep["delta_g%d" % i] = _cmp(g, P, bound, mask=mask)
            _, z = c.ws(15, i, c.T(i))
            _, mu = c.ws(16, i, c.T(i))
            _, rstd = c.ws(17, i, c.T(i))
            gam, _ = c.tensor(_ln_idx(nn, i), 0)
            dz64, lb = _ln_bwd(g, z, mu, rstd, gam)
            rep["ln_bwd%d" % i] = _ratio(np.abs(d_i(c, i) - dz64), lb)
            dz1, _ = _ln_bwd(g, z, mu, rstd, np.ones_like(gam))
            neg.setdefault("gamma_omitted", []).append(_ratio(np.abs(d_i(c, i) - dz1), lb))
            LEDGER["stages"].add("ln_bwd")
            got, want_noalpha, want_noD = g, P1, (noD if inter else None)
        else:
            got = d_i(c, i)
            rep["delta%d" % i] = _cmp(got, P, bound, mask=mask)
            want_noalpha, want_noD = P1, (noD if inter else None)
        LEDGER["stages"].add("delta")
        if alpha != 1.0:
            wa = want_noalpha + (P2 / alpha if inter else 0.0)
            neg.setdefault("alpha_omitted", []).append(_cmp(got, wa, bound, mask=mask))
        if inter:
            neg.setdefault("D_aux_dropped", []).append(_cmp(got, want_noD, bound, mask=mask))


def d_i(c, i):
    return c.ws(7, i, c.T(i))[1]


def _cond_backward(c, rep, neg, m, dd, d, W, Wp, alpha):
    """D'_m = delta_{m+1} W_{m+1} and dP = D'_m W_c recomputed at the step's plans and checked; dA = softmax backward
    (P, dP) + D_aux; the delta alpha [X_m > 0] (D'_m + dA W_{N+1}); dW_c = D'_m^T P, db_c = column sums of D'_m."""
    nn = c.nn
    N, H, K, R = nn.numLayers, nn.layerSize, nn.outputDim, c.R(m)
    assert not (nn.subsample > 1 and m + 1 == nn.subsampleLayer)
    n_out = d.shape[1]
    hm = _hook(nn, 7, m)
    # the step writes D'_m into map m's delta buffer, or into the dh pair at an LSTM layer; both are 256-byte aligned
    # areas of the workspace, and the plans below depend on a pointer only through its alignment
    delta_ptr = nn._ws[hm[0]:].data_ptr()
    plan = _plan(0, 0, R, H, n_out, dd.data_ptr(), n_out, Wp, H)
    cb = _note("delta", plan, n_out)
    dm_dev, Dm = _recompute(0, 0, R, H, n_out, 1.0, dd.data_ptr(), n_out, Wp, H, step_plan=plan)
    P, S = _mm(d, W)
    rep["cond_Dm"] = _cmp(Dm, P, cb * U * S)
    Wc, Wcp = c.tensor(len(nn.stack) - 1, 0)
    plan_p = _plan(0, 0, R, K, H, delta_ptr, H, Wcp, K)
    assert _plan(0, 0, R, K, H, dm_dev.data_ptr(), H, Wcp, K) == plan_p
    cbp = _note("cond", plan_p, H)
    dp_dev, dP = _recompute(0, 0, R, K, H, 1.0, dm_dev.data_ptr(), H, Wcp, K, step_plan=plan_p)
    Pp, Sp = _mm(Dm, Wc)
    rep["cond_dP"] = _cmp(dP, Pp, cbp * U * Sp)
    Pdev, Pm = c.ws(13, 0, c.T(m))
    _, Da = c.ws(9, 0, c.T(m))
    dAd, dA = c.ws(14, 0, c.T(m))
    P64, D64 = Pm.astype(np.float64), dP.astype(np.float64)
    want = P64 * (D64 - (P64 * D64).sum(axis=1, keepdims=True)) + Da
    mag = P64 * (np.abs(D64) + (P64 * np.abs(D64)).sum(axis=1, keepdims=True))
    rep["cond_dA"] = _ratio(np.abs(dA - want), (4 + 2 * K) * U * (mag + np.abs(Da)) + 1e-45)
    # the delta: alpha dA W_{N+1} + alpha D'_m, masked by X_m unless m is temporal (then the BPTT overwrote it)
    Wo, Wop = c.tensor(N, 0)
    plan_d = _plan(0, 0, R, H, K, dAd.data_ptr(), K, Wop, H)
    cbd = _note("cond", plan_d, K)
    if not _temporal(nn, m):
        xm, _ = c.act(m)
        P3, S3 = _mm(dA, Wo, alpha)
        want = P3 + alpha * Dm.astype(np.float64)
        bound = cbd * U * (S3 + abs(alpha) * np.abs(Dm))
        got = d_i(c, m)
        rep["cond_delta"] = _cmp(got, want, bound, mask=xm)
        if alpha != 1.0:
            neg.setdefault("alpha_omitted", []).append(_cmp(got, want / alpha, bound, mask=xm))
        LEDGER["stages"].add("cond_delta")
    elif nn.cell == "lstm":                     # dh = D'_m + dA W_{N+1}, no mask: the BPTT starts from it
        dh_d, dh = _recompute(0, 0, R, H, K, 1.0, dAd.data_ptr(), K, Wop, H, beta=1.0, c0=Dm, step_plan=plan_d)
        P3, S3 = _mm(dA, Wo)
        rep["cond_dh_lstm"] = _cmp(dh, P3 + Dm.astype(np.float64), cbd * U * (S3 + np.abs(Dm)))
        neg.setdefault("D_aux_dropped", []).append(_cmp(dh, Dm.astype(np.float64), cbd * U * (S3 + np.abs(Dm))))
        LEDGER["stages"].add("cond_dh_lstm")
        _lstm_bptt(c, m, dh_d, dh, rep, neg)
    # dW_c = D'_m^T P (beta 0 in a first call), db_c = column sums of D'_m
    gW = nn.grad[len(nn.stack) - 1][0].cpu().numpy()
    gb = nn.grad[len(nn.stack) - 1][1].cpu().numpy().reshape(-1)
    plan_w = _plan(1, 0, H, K, R, delta_ptr, H, Pdev.data_ptr(), K)
    cbw = _note("cond", plan_w, R)
    Pw, Sw = _mm(Dm.T, Pm)
    rep["cond_dWc"] = _cmp(gW, Pw, cbw * U * Sw)
    cplan = _colsum_plan(R, H, delta_ptr)
    Dm64 = Dm.astype(np.float64)
    rep["cond_dbc"] = _ratio(np.abs(gb - Dm64.sum(axis=0)), _colsum_bound(np.abs(Dm64).sum(axis=0), cplan))
    LEDGER["stages"].update(("cond_Dm", "cond_dP", "cond_dA", "cond_dWc", "cond_dbc"))


def _maps(c, rep):
    """Every map's dW, db from the step's delta and the input the map read (part (c)), dW_{N+1} and db_{N+1} with the
    intermediate term D^T X_m (D = D_aux, or dA when self-conditioned)."""
    nn = c.nn
    N, H, K = nn.numLayers, nn.layerSize, nn.outputDim
    for j in range(1, N + 2):
        h = _hook(nn, 7, j)
        if h is None:
            rep["maps%d" % j] = "overwritten"
            continue
        dd, d = c.ws(7, j, c.T(j))
        rows, R = d.shape[1], c.R(j)
        x, xp = c.map_input(j)
        cols = x.shape[1]
        gW = nn.grad[j - 1][0].cpu().numpy().astype(np.float64)
        gb = nn.grad[j - 1][1].cpu().numpy().reshape(-1).astype(np.float64)
        plan = _gemm_plan(rows, cols, R, dd.data_ptr(), rows, xp, cols)
        cb = _note("dW", plan, R)
        P, S = _mm(d.T, x)
        bound = cb * U * S
        d64 = d.astype(np.float64)
        want_b = d64.sum(axis=0)
        bound_b = _colsum_bound(np.abs(d64).sum(axis=0), _colsum_plan(R, rows, dd.data_ptr()))
        if j == N + 1 and nn.interLayer:
            m = nn.interLayer
            Dd, D = c.ws(14 if nn.selfCondition else 9, 0, c.T(m))
            xm, xmp = c.act(m)
            plan2 = _gemm_plan(K, H, c.R(m), Dd.data_ptr(), K, xmp, H)
            cb2 = _note("head", plan2, c.R(m))
            P2, S2 = _mm(D.T, xm)
            bound = bound + cb2 * U * (S2 + np.abs(P))
            P = P + P2
            D64 = D.astype(np.float64)
            bound_b = bound_b + _colsum_bound(np.abs(D64).sum(axis=0), _colsum_plan(c.R(m), K, Dd.data_ptr()), want_b)
            want_b = want_b + D64.sum(axis=0)
            LEDGER["stages"].update(("head_dW", "head_db"))
        rep["maps%d" % j] = dict(dW=_ratio(np.abs(gW - P), bound), db=_ratio(np.abs(gb - want_b), bound_b),
                                 kernel=plan["kernel"])
        LEDGER["stages"].update(("maps_dW", "maps_db"))


@pytest.mark.parametrize("name", list(NETS))
def test_every_stage_of_the_step_from_its_own_inputs(name, cuda):
    torch = cuda
    c = NETS[name]
    nn = _net(c)
    lens, (datas, labelss) = _batches(c, 41)
    batch = nn.swap_batches().pack(datas, labelss).upload()
    nn.dropoutShard = SHARD
    nn.costAndGradDevice(batch, want_probs=True)
    torch.cuda.synchronize()
    call = Call(nn, batch, lens, labelss)
    rep, neg = {}, {}
    reached, LEDGER["stages"] = LEDGER["stages"], set()
    try:
        _forward(call, rep, neg)
        _backward(call, rep, neg)
        _maps(call, rep)
        if nn.interLayer:
            _daux(call, rep, neg)
    finally:
        LEDGER["missing"][name] = sorted(_want(nn) - LEDGER["stages"])
        LEDGER["stages"] |= reached
    LEDGER["rec"][name] = sorted(_rec_missing(call))
    ratios = [v for v in rep.values() if isinstance(v, float)]
    ratios += [v[k] for v in rep.values() if isinstance(v, dict) for k in ("ratio", "dW", "db") if k in v]
    ratios += [x for k, v in rep.items() if k.startswith(("rec", "lstm_fwd")) for x in v.values()]
    negs = {k: min(v) for k, v in neg.items() if v and all(x is not None for x in v)}
    print(json.dumps({"step_stages_" + name: dict(stages=rep, negative_controls=negs)}))
    assert max(ratios) <= 1.0, {k: v for k, v in rep.items() if (v if isinstance(v, float) else 0) > 1.0 or
                                (isinstance(v, dict) and max(v.get("ratio", 0), v.get("dW", 0), v.get("db", 0)) > 1)}
    assert all(v >= NEG for v in negs.values()), negs
    kw = c["kw"]
    if kw.get("dropout"):
        assert "alpha_omitted" in negs or "alpha_fwd" in negs
    if kw.get("interLayer") and not kw.get("selfCondition") and not _temporal(nn, kw["interLayer"]):
        assert "D_aux_dropped" in negs
    if kw.get("weightNoise"):
        assert "clean_params" in negs
    if kw.get("freqMasks"):
        assert "raw_feats" in negs
    if kw.get("layerNorm"):
        assert "gamma_omitted" in negs
    if kw.get("interLayer") and kw.get("subsample", 1) > 1 and kw["interLayer"] >= kw["subsampleLayer"]:
        assert "full_rate_lens" in negs
    if kw.get("cell") == "lstm" and not kw.get("unidirectional"):
        assert "other_direction_U" in negs
    if kw.get("cell") == "lstm" and kw.get("weightNoise"):
        assert "clean_U" in negs
    if kw.get("peephole"):
        assert "P_omitted" in negs and "dp_o_with_c_prev" in negs
    if kw.get("zoneoutCell"):
        assert "zoneout_draw_of_next_step" in negs and "zoneout_numbered_by_u" in negs
    if kw.get("temporalLayer") and not kw.get("unidirectional"):
        assert "direction_1_unshifted" in negs
    if kw.get("cell") == "lstm" and kw.get("interLayer") == kw.get("temporalLayer"):
        assert "D_aux_dropped" in negs
    assert not LEDGER["missing"][name], LEDGER["missing"][name]
    assert not LEDGER["rec"][name], "no recurrent gradient check at layers %s" % LEDGER["rec"][name]


def _rec_missing(call):
    """The temporal layers of the call's net whose recurrent gradients were not checked."""
    nn = call.nn
    return {i for i in range(1, nn.numLayers + 1) if _temporal(nn, i)} - call.rec_done


def test_every_path_was_reached(cuda):
    """Both contraction kernels in the forward maps, the deltas, the weight gradients and the head / conditioning
    contractions; split-K in a forward map (the stacked map of uni_h256_sub2_splitk); all three ReLU sweep families
    (generic, cluster, tensor-core at H = 1024); the LSTM sweep with U in registers and re-read; every stage kind,
    every net the stage kinds of its features, and every temporal layer its recurrent gradients."""
    missing = sorted(WANT_STAGES - LEDGER["stages"])
    kernels = {k: sorted(v) for k, v in LEDGER["kernels"].items()}
    print(json.dumps({"step_stages_ledger": dict(kernels=kernels, splitk=sorted(LEDGER["splitk"]),
                                                 sweeps=sorted(LEDGER["sweeps"]), lstm_ki=sorted(LEDGER["lstm_ki"]),
                                                 stages=sorted(LEDGER["stages"]))}))
    assert not missing, missing
    for kind in ("fwd", "delta", "dW", "head", "cond"):
        assert LEDGER["kernels"].get(kind) == {0, 1}, (kind, kernels)
    assert "fwd" in LEDGER["splitk"], LEDGER["splitk"]
    assert {"generic", "cluster", "tensor-core"} <= LEDGER["sweeps"], LEDGER["sweeps"]
    assert 0 in LEDGER["lstm_ki"] and LEDGER["lstm_ki"] - {0}, LEDGER["lstm_ki"]
    assert len(LEDGER["missing"]) == len(NETS) and not any(LEDGER["missing"].values()), LEDGER["missing"]
    assert len(LEDGER["rec"]) == len(NETS) and not any(LEDGER["rec"].values()), LEDGER["rec"]
