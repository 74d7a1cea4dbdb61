"""stack_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of a net with a block of stacked temporal layers.

The one-temporal-layer restatement (oracle/brnn_oracle.py) is pinned to the reference's own rnnetcpu.py and stays as it
is.  This class generalises its loops to numTemporal = k contiguous temporal layers temporalLayer .. temporalLayer+k-1,
each a clipped-ReLU recurrence with its own matrices (brnnet.py:143-153 bi-directional, rnnet.py:112-116
uni-directional), back-propagated layer by layer with the BPTT of brnnet.py:207-233 / rnnet.py:162-177.  Layers outside
the block are the ReLU hidden layers and the linear output layer of the reference.  Stack order and np.random draw
order are those of nnets.brnnet.NNet: [W1,b1] .. [W_{N+1},b_{N+1}], then per temporal layer [Wtf_j,dummy] [Wtb_j,dummy]
(uni-directional [Wt_j,dummy]).  With k = 1 it computes what brnn_oracle.NNet computes (tests/test_stack_cpu.py), and
for k > 1 it is checked by central finite differences.  L2 adds reg*W to every weight matrix, recurrent ones included,
as the library does.  The CTC half is brnn_oracle's (pinned to the reference's ctc_fast.pyx)."""
import numpy as np

from oracle import brnn_oracle


class StackNet:
    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal=1, reg=0.0,
                 dtype=np.float64, allow_top_temporal=False, round_f32=True, unidirectional=False):
        hi = numLayers + 1 if allow_top_temporal else numLayers
        assert 1 <= temporalLayer and temporalLayer + max(1, numTemporal) - 1 < hi, "the block must fit"
        self.inputDim, self.outputDim, self.layerSize, self.numLayers = inputDim, outputDim, layerSize, numLayers
        self.maxBatch, self.reg, self.dtype, self.round_f32 = maxBatch, reg, dtype, round_f32
        self.temporalLayer, self.numTemporal = temporalLayer, max(1, numTemporal)
        self.unidirectional = unidirectional
        self.nrec = 1 if unidirectional else 2
        self.maxAct = 20.0
        self.regcost = 0.0

    def temporal(self, i):
        return self.temporalLayer <= i < self.temporalLayer + self.numTemporal

    def rec(self, j):
        """Stack indices of the recurrent matrices of temporal layer j (0-based within the block)."""
        base = self.numLayers + 1 + j * self.nrec
        return base, (None if self.unidirectional else base + 1)

    def initParams(self):
        sizes = [self.inputDim] + [self.layerSize] * self.numLayers + [self.outputDim]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(sizes[:-1], sizes[1:])]
        self.stack = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))]
                      for n, m, s in zip(sizes[:-1], sizes[1:], scales)]
        scale = np.sqrt(6) / np.sqrt(self.layerSize * 2)
        for _ in range(self.numTemporal):
            for _ in range(self.nrec):
                w = 2 * scale * np.random.rand(self.layerSize, self.layerSize) - scale
                self.stack.append([w, np.zeros((1, 1))])
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in self.stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    def _softmax(self, logits):
        z = logits - logits.max(axis=0)[None, :]
        e = np.exp(z)
        probs = e / e.sum(axis=0)[None, :]
        return probs.astype(np.float32) if self.round_f32 else probs

    def forward(self, data):
        """Returns (hActs [data, h_1 .. h_{N+1}], Fors, Backs, probs); Fors / Backs hold one array per temporal layer
        (Backs None when uni-directional)."""
        T = data.shape[1]
        hActs = [np.asarray(data, dtype=self.dtype)]
        Fors, Backs = [], []
        for i in range(1, self.numLayers + 2):
            w, b = self.stack[i - 1]
            h = w.dot(hActs[i - 1]) + b
            if self.temporal(i):
                f_idx, b_idx = self.rec(i - self.temporalLayer)
                wtf = self.stack[f_idx][0]
                For = h.copy()
                For[:, 0] = np.clip(For[:, 0], 0.0, self.maxAct)
                for t in range(1, T):
                    For[:, t] = np.clip(For[:, t] + wtf.dot(For[:, t - 1]), 0.0, self.maxAct)
                Fors.append(For)
                if self.unidirectional:
                    h = For
                    Backs.append(None)
                else:
                    wtb = self.stack[b_idx][0]
                    Back = h.copy()
                    Back[:, T - 1] = np.clip(Back[:, T - 1], 0.0, self.maxAct)
                    for t in range(1, T):
                        Back[:, T - t - 1] = np.clip(Back[:, T - t - 1] + wtb.dot(Back[:, T - t]), 0.0, self.maxAct)
                    Backs.append(Back)
                    h = For + Back
            elif i <= self.numLayers:
                h = np.maximum(h, 0.0)
            hActs.append(h)
        return hActs, Fors, (None if self.unidirectional else Backs), self._softmax(hActs[-1])

    def costAndGradGiven(self, data, labels, hActs, Fors, Backs):
        """Back-propagation through GIVEN activations (h_1 .. h_{N+1}, For_j, Back_j), e.g. the GPU's: the masks are
        then the implementation's own (see brnn_oracle.NNet.costAndGradGiven)."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(h, dtype=dt) for h in hActs]
        Fors = [np.asarray(f, dtype=dt) for f in Fors]
        Backs = None if Backs is None else [np.asarray(b, dtype=dt) for b in Backs]
        return self.costAndGrad(data, labels, _given=(hActs, Fors, Backs, self._softmax(hActs[-1])))

    def costAndGrad(self, data, labels, _given=None):
        hActs, Fors, Backs, probs = self.forward(data) if _given is None else _given
        T = data.shape[1]
        dt = self.dtype
        cost, deltas, skip = brnn_oracle._ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                                   np.asarray(labels, dtype=np.int32))
        grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        if self.reg > 0:
            self.regcost = sum((self.reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2)) for w, _ in self.stack)
            cost = cost + self.regcost
        if skip:
            self.grad = grad
            return cost, grad, skip
        deltasIn = (deltas.astype(np.float32) if self.round_f32 else deltas).astype(dt)
        for i in range(self.numLayers, -1, -1):
            w = self.stack[i][0]
            grad[i][0] = deltasIn.dot(hActs[i].T)
            grad[i][1] = deltasIn.sum(axis=1)[:, None]
            if i == 0:
                break
            deltasOut = w.T.dot(deltasIn)
            if self.temporal(i):
                j = i - self.temporalLayer
                f_idx, b_idx = self.rec(j)
                For = Fors[j]
                mF = ((For > 0.0) & (For < self.maxAct)).astype(dt)
                wtf = self.stack[f_idx][0]
                pre = deltasOut
                dFor = pre.copy()
                dFor[:, T - 1] *= mF[:, T - 1]
                for t in range(T - 1, 0, -1):
                    dFor[:, t - 1] += wtf.T.dot(dFor[:, t])
                    dFor[:, t - 1] *= mF[:, t - 1]
                grad[f_idx][0] = dFor[:, 1:T].dot(For[:, 0:T - 1].T)
                deltasOut = dFor
                if not self.unidirectional:
                    Back = Backs[j]
                    mB = ((Back > 0.0) & (Back < self.maxAct)).astype(dt)
                    wtb = self.stack[b_idx][0]
                    dBack = pre.copy()
                    dBack[:, 0] *= mB[:, 0]
                    for t in range(1, T):
                        dBack[:, t] += wtb.T.dot(dBack[:, t - 1])
                        dBack[:, t] *= mB[:, t]
                    grad[b_idx][0] = dBack[:, 0:T - 1].dot(Back[:, 1:T].T)
                    deltasOut = dFor + dBack
            else:
                deltasOut = deltasOut * (hActs[i] > 0.0)
            deltasIn = deltasOut
        if self.reg > 0:
            for g, (w, _) in zip(grad, self.stack):
                g[0] += self.reg * w
        self.grad = grad
        return cost, grad, skip

    def costAndGradBatch(self, datas, labelss):
        """Per-utterance gradients summed (a skipped utterance adds nothing), the L2 term added once."""
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
            for (w, _), (tw, _) in zip(self.stack, tot):
                self.regcost += (reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                tw += reg * w
        self.grad = tot
        return np.array(costs), self.grad, np.array(skips)
