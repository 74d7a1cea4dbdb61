"""oracle/brnn_oracle.py -- TEST INFRASTRUCTURE ONLY (checker + CPU baseline "port").

NumPy restatement of the reference BRNN training step, per utterance, following line by line
  ctc_fast/nnets/brnnet.py:10-32   (ctor; temporalLayer rule; maxAct = 20)
  ctc_fast/nnets/brnnet.py:34-86   (initParams: shapes and np.random draw order)
  ctc_fast/nnets/brnnet.py:117-173 (forward; clipped-ReLU recurrences; softmax)
  ctc_fast/nnets/brnnet.py:175-249 (CTC, L2 cost, back-prop / BPTT, L2 grad)
  ctc_fast/nnets/brnnet.py:251-256 (updateParams)
  ctc_fast/sgd.py:57-167           (Nesterov step, global-norm clip)
cross-checked against the reference's own NumPy BRNN
  ctc_fast/debug-utils/rnnetcpu.py:54-150 (same math without the 20-clip / L2).

PINNED (round 2): tests/golden/rnnetcpu_ref.npz holds inputs/outputs of the reference's own
rnnetcpu.RNNet.costAndGrad executed in the authoring container (tests/golden/gen_rnnetcpu_ref.py: the file as
it lies in the reference checkout, print/xrange/tabs converted mechanically, CTC = oracle/_ref); configured as that file
computes (float64, no clip, no float32 hand-offs, no L2) this restatement reproduces cost and all gradients of
5 shapes to 1e-12 (tests/test_oracle.py::test_brnn_restatement_pinned_to_reference_rnnetcpu).
What brnnet.py adds on top of rnnetcpu.py -- the 20.0 clip / within() mask, the float32 hand-offs and L2 -- runs
inside cudamat in the reference (fork github.com/awni/cudamat, no pinned version, source absent from
the reference checkout); for those three additions the restatement follows the call sites and is checked by finite
differences only.
Semantics adopted from the call sites and rnnetcpu.py:
  mvdot_col_slice(W,src,i,dst,j,beta=1): dst[:,j] = beta*dst[:,j] + W.dot(src[:,i])
  minmax(lo,hi,col=c): clamp column c into [lo,hi]
  within(lo,hi): 1.0 where lo < x < hi else 0.0   (== sign() mask of rnnetcpu.py:125-126 below 20)
  mult_slice(c,M,c): self[:,c] *= M[:,c]
  sign(): 1 for x>0, 0 for x==0 (activations are >= 0 after ReLU)
The CTC half IS pinned: it calls oracle/_ref (the unmodified ctc_fast.pyx) when built, else the
C restatement oracle/ctc_oracle.c, which is itself verified bit-for-bit against oracle/_ref.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.
"""
import numpy as np

from . import ctc_oracle as _ctc


def _ctc_loss(probs64_F, labels, use_ref=True):
    if use_ref and _ctc.ref_module() is not None:
        return _ctc.ref_ctc_loss(probs64_F, labels, 0)
    return _ctc.ctc_loss(probs64_F, labels, 0)


class NNet:
    """Same constructor and attributes as brnnet.NNet (brnnet.py:10-32).  `dtype` selects the
    arithmetic of the dense part: float32 mirrors cudamat, float64 is the tight checker."""

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, train=True,
                 temporalLayer=-1, reg=0.0, dtype=np.float64, allow_top_temporal=False,
                 round_f32=True, unidirectional=False):
        self.outputDim, self.inputDim = outputDim, inputDim
        self.layerSize, self.numLayers = layerSize, numLayers
        self.layerSizes = [layerSize] * numLayers
        self.maxBatch, self.train, self.reg = maxBatch, train, reg
        self.regcost = 0.0
        self.dtype = dtype
        # round_f32: mirror the reference's float32 hand-offs (probs D2H :170, deltas H2D :188);
        # switch off only for finite-difference checks of this restatement itself
        self.round_f32 = round_f32
        # brnnet.py:27-30; allow_top_temporal is the documented extension temporalLayer==numLayers
        hi = numLayers + 1 if allow_top_temporal else numLayers
        self.temporalLayer = -1 if (temporalLayer <= 0 or temporalLayer >= hi) else temporalLayer
        self.maxAct = 20.0
        # unidirectional: the restatement of nnets/rnnet.py:8-191 (one recurrent matrix, forward in time only);
        # with temporalLayer=-1 either setting is nnets/nnet.py:57-113 (same loops without the temporal branch)
        self.unidirectional = unidirectional
        self.nrec = 0 if self.temporalLayer <= 0 else (1 if unidirectional else 2)

    def initParams(self):
        # brnnet.py:38-41 then :66-70 -- identical draw order from the global np.random stream
        sizes = [self.inputDim] + self.layerSizes + [self.outputDim]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(sizes[:-1], sizes[1:])]
        self.stack = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))]
                      for n, m, s in zip(sizes[:-1], sizes[1:], scales)]
        if self.temporalLayer > 0:
            scale = np.sqrt(6) / np.sqrt(self.layerSize * 2)
            wtf = 2 * scale * np.random.rand(self.layerSize, self.layerSize) - scale
            self.stack.append([wtf, np.zeros((1, 1))])
            if not self.unidirectional:                                   # rnnet.py:57-61: a single wt
                wtb = 2 * scale * np.random.rand(self.layerSize, self.layerSize) - scale
                self.stack.append([wtb, np.zeros((1, 1))])
        # cudamat stores float32 (cm.CUDAMatrix(w) converts): round the float64 draws once
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in self.stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    def paramCount(self):
        return int(sum(w.size + b.size for w, b in self.stack))

    def forward(self, data):
        """brnnet.py:136-168.  Returns (hActs list, For, Back, probs) with probs float32-rounded."""
        dt = self.dtype
        T = data.shape[1]
        stack = self.stack[:-self.nrec] if self.nrec else self.stack
        hActs = [np.asarray(data, dtype=dt)]
        For = Back = None
        i = 1
        for w, b in stack:
            h = w.dot(hActs[i - 1]) + b                                    # :140-141
            if i == self.temporalLayer and self.unidirectional:           # rnnet.py:112-116
                wt = self.stack[-1][0]
                For = h.copy()
                For[:, 0] = np.clip(For[:, 0], 0.0, self.maxAct)
                for t in range(1, T):
                    For[:, t] = np.clip(For[:, t] + wt.dot(For[:, t - 1]), 0.0, self.maxAct)
                h = For
            elif i == self.temporalLayer:                                 # :143-153
                wtf, wtb = self.stack[-2][0], self.stack[-1][0]
                For, Back = h.copy(), h.copy()
                For[:, 0] = np.clip(For[:, 0], 0.0, self.maxAct)
                Back[:, T - 1] = np.clip(Back[:, T - 1], 0.0, self.maxAct)
                for t in range(1, T):
                    For[:, t] = np.clip(For[:, t] + wtf.dot(For[:, t - 1]), 0.0, self.maxAct)
                    Back[:, T - t - 1] = np.clip(Back[:, T - t - 1] + wtb.dot(Back[:, T - t]), 0.0, self.maxAct)
                h = For + Back
            if i <= self.numLayers and i != self.temporalLayer:           # :155-157
                h = np.maximum(h, 0.0)
            hActs.append(h)
            i += 1
        z = hActs[-1] - hActs[-1].max(axis=0)[None, :]                    # :161-168
        e = np.exp(z)
        probs = e / e.sum(axis=0)[None, :]
        return hActs, For, Back, (probs.astype(np.float32) if self.round_f32 else probs)

    def costAndGradGiven(self, data, labels, hActs, For, Back):
        """Checker-only: back-propagation (brnnet.py:175-249) THROUGH GIVEN ACTIVATIONS -- hActs[1..N+1] (the last
        entry the pre-softmax outputs), For, Back, as the implementation under test computed them, widened to this
        net's dtype.  The ReLU / clip masks are then the implementation's own, so the comparison of the gradients
        measures its backward arithmetic and is blind to the mask flips that float32 noise in the forward pass
        causes (profiles/kink_sensitivity_r2.txt)."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(h, dtype=dt) for h in hActs]
        z = hActs[-1] - hActs[-1].max(axis=0)[None, :]
        e = np.exp(z)
        probs = e / e.sum(axis=0)[None, :]
        probs = probs.astype(np.float32) if self.round_f32 else probs
        return self.costAndGrad(data, labels, _given=(hActs, None if For is None else np.asarray(For, dtype=dt),
                                                       None if Back is None else np.asarray(Back, dtype=dt), probs))

    def costAndGrad(self, data, labels=None, sentence=None, _given=None):
        hActs, For, Back, probs = self.forward(data) if _given is None else _given
        if not self.train:
            return probs                                                  # :171-173
        T = data.shape[1]
        dt = self.dtype
        # :175 -- the reference widens the float32 probs to float64 for the Cython CTC
        cost, deltas, skip = _ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                       np.asarray(labels, dtype=np.int32))
        if self.reg > 0:                                                  # :177-183
            self.regcost = 0.0
            for w, b in self.stack:
                rc = (self.reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                self.regcost += rc
                cost = cost + rc
        if skip:
            return cost, self.grad, skip                                  # :185-186
        if self.nrec == 1:
            stack, grad = self.stack[:-1], self.grad[:-1]
            wtf = self.stack[-1][0]
        elif self.nrec == 2:
            stack, grad = self.stack[:-2], self.grad[:-2]
            wtf, wtb = self.stack[-2][0], self.stack[-1][0]
        else:
            stack, grad = self.stack, self.grad
        deltasIn = (deltas.astype(np.float32) if self.round_f32 else deltas).astype(dt)  # :188
        i = self.numLayers
        for w, b in reversed(stack):                                      # :191-243
            grad[i][0] = deltasIn.dot(hActs[i].T)                         # :196
            if self.reg > 0:
                grad[i][0] = grad[i][0] + self.reg * w                    # :197-198
            grad[i][1] = deltasIn.sum(axis=1)[:, None]                    # :200
            deltasOut = None
            if i > 0:
                deltasOut = w.T.dot(deltasIn)                             # :203-204
            if i == self.temporalLayer and self.unidirectional:           # rnnet.py:162-177
                mF = ((For > 0.0) & (For < self.maxAct)).astype(dt)
                dFor = deltasOut.copy()
                dFor[:, T - 1] *= mF[:, T - 1]
                for t in range(T - 1, 0, -1):
                    dFor[:, t - 1] += wtf.T.dot(dFor[:, t])
                    dFor[:, t - 1] *= mF[:, t - 1]
                self.grad[-1][0] = dFor[:, 1:T].dot(For[:, 0:T - 1].T)    # rnnet.py:173-174 (deltaTemp = delta shifted by one)
                deltasOut = dFor
            elif i == self.temporalLayer:                                 # :207-233
                mF = ((For > 0.0) & (For < self.maxAct)).astype(dt)       # within(0,maxAct)
                mB = ((Back > 0.0) & (Back < self.maxAct)).astype(dt)
                dFor, dBack = deltasOut.copy(), deltasOut.copy()
                dFor[:, T - 1] *= mF[:, T - 1]
                dBack[:, 0] *= mB[:, 0]
                for t in range(1, T):
                    dFor[:, T - t - 1] += wtf.T.dot(dFor[:, T - t])
                    dBack[:, t] += wtb.T.dot(dBack[:, t - 1])
                    dFor[:, T - t - 1] *= mF[:, T - t - 1]
                    dBack[:, t] *= mB[:, t]
                self.grad[-2][0] = dFor[:, 1:T].dot(For[:, 0:T - 1].T)    # :227-228
                self.grad[-1][0] = dBack[:, 0:T - 1].dot(Back[:, 1:T].T)  # :229-230
                deltasOut = dFor + dBack                                  # :233
            if i > 0 and i != self.temporalLayer:                         # :235-237
                deltasOut = deltasOut * (hActs[i] > 0.0)
            deltasIn = deltasOut
            i -= 1
        if self.reg > 0 and self.nrec == 2:                               # :244-247
            self.grad[-2][0] = self.grad[-2][0] + self.reg * wtf
            self.grad[-1][0] = self.grad[-1][0] + self.reg * wtb
        return cost, self.grad, skip

    def costAndGradBatch(self, datas, labelss):
        """Minibatch semantics of the new build: per-utterance steps of the reference summed
        (un-normalised, cf. ctc/nnet.py:193-195); a skipped utterance contributes zero gradient.
        The L2 term is added once per batch."""
        reg, self.reg = self.reg, 0.0
        tot = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        costs, skips = [], []
        for d, l in zip(datas, labelss):
            c, g, s = self.costAndGrad(d, l)
            costs.append(c)
            skips.append(bool(s))
            if not s:
                for (tw, tb), (gw, gb) in zip(tot, g):
                    tw += gw
                    tb += gb
        self.reg = reg
        self.regcost = 0.0
        if reg > 0:
            for (w, b), (tw, tb) in zip(self.stack, tot):
                self.regcost += (reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                tw += reg * w
        self.grad = tot
        return np.array(costs), self.grad, np.array(skips)

    def updateParams(self, scale, update):
        for (w, b), (dw, db) in zip(self.stack, update):                  # :251-256
            w += scale * dw
            b += scale * db


def sgd_step(model, velocity, grad, it, alpha, momentum, maxGNorm=1500.0):
    """sgd.py:64-74,103-107,130-161 given the gradient evaluated at the look-ahead point.
    The caller brackets costAndGrad with updateParams(+mom)/(-mom) as sgd.py:93,100 do.
    Returns (gnorm, mom)."""
    mom = 0.5 if it <= 10 else momentum
    gnorm = np.sqrt(sum(float(np.sum(dw.astype(np.float64) ** 2)) + float(np.sum(db.astype(np.float64) ** 2))
                        for dw, db in grad))
    alph = alpha
    if gnorm > maxGNorm:
        alph *= maxGNorm / gnorm
    for (vw, vb), (dw, db) in zip(velocity, grad):
        vw *= mom
        vb *= mom
        vw += -alph * dw
        vb += -alph * db
    model.updateParams(1.0, velocity)
    return gnorm, mom
