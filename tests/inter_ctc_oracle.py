"""inter_ctc_oracle.py -- TEST INFRASTRUCTURE ONLY: the float64 restatement of a net trained with an intermediate CTC
loss (include/ctcb200.h: interLayer), built on tests/net_oracle.Net through tests/peephole_oracle.PeepholeNet, so the
loss composes with peepholes (peephole defaults to False here, and PeepholeNet is then Net).

Hidden layer m's output X_m (as map m + 1 sees it) goes through the output map: A = W_{N+1} X_m + b_{N+1}, on layer m's
own frames; nll_aux is the CTC loss of softmax(A).  The objective is nll_main + lambda nll_aux.  Because the gradient
of that sum is the sum of the gradients, the restatement needs no new back-propagation: the intermediate term is the
gradient of the HEAD NET, the same class with hidden layers 1..m (their temporal layers, normalisation, dropout masks and
subsampling, when it starts at or below m) and the output map W_{N+1}, b_{N+1} on top.  Its stack holds the very arrays
of the full net's, so it computes X_m as the full net does, bit for bit, and its gradient, times lambda (the float32 the
library is given), is added tensor by tensor.  Each CTC skips on its own.

InterNet.costAndGrad returns (main cost, gradient of the objective, main skip), as net_check.compare expects, and
leaves the intermediate nll and skip in interCost / interSkip; objective() is main + lambda nll_aux.  With
interLayer = 0 it is Net (or PeepholeNet)."""
import numpy as np

from peephole_oracle import PeepholeNet


class InterNet(PeepholeNet):
    def __init__(self, *args, peephole=False, interLayer=0, interWeight=0.0, **kw):
        PeepholeNet.__init__(self, *args, peephole=peephole, **kw)
        self._kw = dict(kw, peephole=peephole)
        self.interLayer, self.interWeight = int(interLayer), float(interWeight)
        if self.interLayer != 0 and not (np.isfinite(self.interWeight) and self.interWeight > 0.0):
            raise ValueError("interLayer=%d needs a finite interWeight > 0" % self.interLayer)
        if self.interLayer == 0 and self.interWeight != 0.0:
            raise ValueError("interWeight=%r needs interLayer >= 1" % (interWeight,))
        if self.interLayer and not 1 <= self.interLayer <= self.numLayers - 1:
            raise ValueError("interLayer %d is not one of the hidden layers 1..%d" % (self.interLayer,
                                                                                    self.numLayers - 1))
        if self.interLayer and self.k > 1 and self.L == self.numLayers + 1:
            raise ValueError("interLayer with subsampling at the output map")
        self.interCost, self.interSkip = 0.0, False

    def lam(self):
        return float(np.float32(self.interWeight))

    # ------------------------------------------------------------------ the head net
    def _keys(self, net, top):
        """Semantic key of every stack index of `net`, whose output map counts as map `top`."""
        keys = [("map", i if i <= net.numLayers else top) for i in range(1, net.numLayers + 2)]
        for j in range(net.numTemporal):
            keys += [("rec", j, d) for d in range(net.nrec)]
        keys += [("ln", i) for i in net.normedLayers()]
        if net.peephole:
            keys += [("peep", j, d) for j in range(net.numTemporal) for d in range(net.nrec)]
        return keys

    def head(self):
        """The head net over the same arrays: hidden layers 1..m and the output map, and the index of each of its
        stack entries in this net's stack."""
        m, tl = self.interLayer, self.temporalLayer
        nt = min(self.numTemporal, m - tl + 1) if self.numTemporal and tl <= m else 0
        kw = dict(self._kw)
        kw.update(temporalLayer=tl if nt else -1, numTemporal=nt, allowTopTemporal=True,
                  subsample=self.k if 0 < self.L <= m else 1, subsampleLayer=self.L if 0 < self.L <= m else 1,
                  dropout=self.dropout, dropoutSeed=self.dropoutSeed, reg=0.0, dtype=self.dtype,
                  round_f32=self.round_f32, unidirectional=self.unidirectional, cell=self.cell,
                  layerNorm=self.layerNorm)
        net = PeepholeNet(self.inputDim, self.outputDim, self.layerSize, m, self.maxBatch, **kw)
        full = {k: t for t, k in enumerate(self._keys(self, self.numLayers + 1))}
        index = [full[k] for k in self._keys(net, self.numLayers + 1)]
        net.stack = [self.stack[t] for t in index]
        net.dropoutStep, net.utt = self.dropoutStep, self.utt
        return net, index

    # ------------------------------------------------------------------ passes
    def costAndGrad(self, data, labels, _given=None):
        if not self.interLayer:
            return PeepholeNet.costAndGrad(self, data, labels, _given)
        if _given is None:
            _given = self.forward(data)
        cost, grad, skip = PeepholeNet.costAndGrad(self, data, labels, _given)
        hActs, temporal, _ = _given
        net, index = self.head()
        m = self.interLayer
        w, b = self.stack[self.numLayers]
        A = w.dot(hActs[m]) + b
        nt = net.numTemporal
        c, g, s = net.costAndGrad(data, labels, _given=(list(hActs[:m + 1]) + [A], temporal[:nt], net._softmax(A)))
        self.interCost, self.interSkip = float(c), bool(s)
        if not s:
            lam = self.lam()
            for t, (gw, gb) in zip(index, g):
                grad[t][0] = grad[t][0] + lam * gw
                grad[t][1] = grad[t][1] + lam * gb
        self.grad = grad
        return cost, grad, skip

    def objective(self, data, labels):
        """nll_main (+ the L2 cost) + lambda nll_aux, the intermediate term left out where its CTC skips."""
        cost, _, _ = self.costAndGrad(data, labels)
        return cost + (0.0 if not self.interLayer or self.interSkip else self.lam() * self.interCost)

    def costAndGradBatch(self, datas, labelss, utts=None):
        """Net's sum, except that an utterance only the main CTC skips still adds its intermediate gradient; leaves
        the per-utterance intermediate nll and skips in interCosts / interSkips."""
        reg, self.reg = self.reg, 0.0
        tot = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        costs, skips, icosts, iskips = [], [], [], []
        for u, (d, l) in enumerate(zip(datas, labelss)):
            self.utt = u if utts is None else utts[u]
            c, g, s = self.costAndGrad(d, l)
            costs.append(c)
            skips.append(bool(s))
            icosts.append(self.interCost)
            iskips.append(self.interSkip)
            for (tw, tb), (gw, gb) in zip(tot, g):
                tw += gw
                tb += gb
        self.reg = reg
        self.regcost = 0.0
        if reg > 0:
            for k in self.weight_indices():
                w = self.stack[k][0]
                self.regcost += (reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                tot[k][0] += reg * w
        self.grad = tot
        self.interCosts, self.interSkips = np.array(icosts), np.array(iskips)
        return np.array(costs), self.grad, np.array(skips)

