"""self_cond_oracle.py -- TEST INFRASTRUCTURE ONLY: the float64 restatement of a self-conditioned CTC net
(include/ctcb200.h: selfCondition), built on tests/inter_ctc_oracle.InterNet.

With A = W_{N+1} X_m + b_{N+1} and P = softmax(A) per frame, map m + 1 (and the frame stacking, when it starts there)
reads X'_m = X_m + W_c P + b_c.  The stack is InterNet's followed by [W_c (H x K), b_c (H x 1)], both 0 without a draw,
not L2-regularised.  The intermediate loss still scores A and does not depend on W_c, so its gradient is InterNet's
head-net term; the main loss needs a real back-propagation through X'_m, which _backward does: Net's backward pass
with, at layer m, D'_m = W_{m+1}^T delta_{m+1} (unstacked), dP = W_c^T D'_m, dA = P (dP - sum_k P_k dP_k),
dW_c = D'_m P^T, db_c = sum_t D'_m, dW_{N+1} += dA X_m^T, db_{N+1} += sum_t dA, and D'_m + W_{N+1}^T dA in place of
D'_m as the delta that layer m's mask, normalisation or BPTT then reads.

costAndGradGiven takes the device's X'_m and P (cond=(X'_m, P), [n][T]) besides the other activations, or, without
cond, givenCond[utt] (a dict a test fills for tests/net_check.compare, which sets utt per utterance).  With
selfCondition=False SelfCondNet is InterNet."""
import numpy as np

import net_oracle
from inter_ctc_oracle import InterNet
from net_oracle import Net, threshold_scale, unstack_frames, stack_frames
from oracle import brnn_oracle


class SelfCondNet(InterNet):
    def __init__(self, *args, selfCondition=False, **kw):
        InterNet.__init__(self, *args, **kw)
        self.selfCondition = bool(selfCondition)
        if self.selfCondition and not self.interLayer:
            raise ValueError("selfCondition=True needs interLayer >= 1")
        self._cond = None       # (X'_m, P) of the device, in costAndGradGiven
        self.givenCond = None   # {utt: (X'_m, P)} of the device

    def shapes(self):
        return InterNet.shapes(self) + ([(self.layerSize, self.outputDim), (self.layerSize, 1)]
                                        if self.selfCondition else [])

    def initParams(self):
        """InterNet's draws; W_c and b_c behind them, 0 without a draw."""
        Net.initParams(self)
        n = len(self.stack) - self.entries() - (1 if self.selfCondition else 0)
        for k in range(n, len(self.stack)):
            self.stack[k][0][...] = 0.0

    # ------------------------------------------------------------------ the conditioning
    def conditioned(self, hActs):
        """(X'_m, P) of the activations hActs (the device's when given)."""
        if self._cond is not None:
            return self._cond
        m, N = self.interLayer, self.numLayers
        P = self._softmax(self.stack[N][0].dot(hActs[m]) + self.stack[N][1]).astype(self.dtype)
        Wc, bc = self.stack[-1]
        return hActs[m] + Wc.dot(P) + bc, P

    def map_input(self, hActs, i):
        if self.selfCondition and i == self.interLayer + 1:
            x = self.conditioned(hActs)[0]
            return stack_frames(x, self.k) if self.stacked(i) else x
        return Net.map_input(self, hActs, i)

    # ------------------------------------------------------------------ passes
    def costAndGradGiven(self, data, labels, hActs, temporal, cond=None):
        if cond is None and self.givenCond is not None:
            cond = self.givenCond[self.utt]
        if cond is not None:
            self._cond = tuple(np.asarray(x, dtype=self.dtype) for x in cond)
        try:
            return Net.costAndGradGiven(self, data, labels, hActs, temporal)
        finally:
            self._cond = None

    def costAndGrad(self, data, labels, _given=None):
        if not self.selfCondition:
            return InterNet.costAndGrad(self, data, labels, _given)
        if _given is None:
            _given = self.forward(data)
        self._dP = {}
        with self._cell():
            cost, grad, skip = self._backward(data, labels, _given)
        for k, dP in self._dP.items():
            grad[k][0] = dP
        # the intermediate term: the head net's gradient, as InterNet's
        hActs, temporal, _ = _given
        net, index = self.head()
        m = self.interLayer
        w, b = self.stack[self.numLayers]
        A = w.dot(hActs[m]) + b
        c, g, s = net.costAndGrad(data, labels, _given=(list(hActs[:m + 1]) + [A], temporal[:net.numTemporal],
                                                         net._softmax(A)))
        self.interCost, self.interSkip = float(c), bool(s)
        if not s:
            lam = self.lam()
            for t, (gw, gb) in zip(index, g):
                grad[t][0] = grad[t][0] + lam * gw
                grad[t][1] = grad[t][1] + lam * gb
        self.grad = grad
        return cost, grad, skip

    def _backward(self, data, labels, given):
        """Net.costAndGrad with the conditioning's backward at layer m (the module docstring)."""
        hActs, temporal, probs = given
        H, dt, m, N = self.layerSize, self.dtype, self.interLayer, self.numLayers
        cost, deltas, skip = brnn_oracle._ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                                   np.asarray(labels, dtype=np.int32))
        grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        if self.reg > 0:
            self.regcost = sum((self.reg / 2.0) * float(np.sum(self.stack[k][0].astype(np.float64) ** 2))
                               for k in self.weight_indices())
            cost = cost + self.regcost
        if skip:
            return cost, grad, skip
        deltasIn = (deltas.astype(np.float32) if self.round_f32 else deltas).astype(dt)
        for i in range(N, -1, -1):
            w = self.stack[i][0]
            grad[i][0] = grad[i][0] + deltasIn.dot(self.map_input(hActs, i + 1).T)
            grad[i][1] = grad[i][1] + deltasIn.sum(axis=1)[:, None]
            if i == 0:
                break
            deltasOut = w.T.dot(deltasIn)
            if self.stacked(i + 1):
                deltasOut = unstack_frames(deltasOut, self.k, hActs[i].shape[1])
            if i == m:
                Xp, P = self.conditioned(hActs)
                Wc = self.stack[-1][0]
                dP = Wc.T.dot(deltasOut)
                dA = P * (dP - (P * dP).sum(axis=0)[None, :])
                grad[-1][0] = deltasOut.dot(P.T)
                grad[-1][1] = deltasOut.sum(axis=1)[:, None]
                grad[N][0] = grad[N][0] + dA.dot(hActs[m].T)
                grad[N][1] = grad[N][1] + dA.sum(axis=1)[:, None]
                deltasOut = deltasOut + self.stack[N][0].T.dot(dA)
            T = deltasOut.shape[1]
            if self.temporal(i):
                j = i - self.temporalLayer
                idx = self.rec(j)
                if self.cell == "lstm":
                    gates, cs, hs = temporal[j]
                    dzs = []
                    for d in range(self.nrec):
                        dz, dU = net_oracle.lstm_direction_bptt(deltasOut, gates[d * 4 * H:(d + 1) * 4 * H], cs[d],
                                                                hs[d], self.stack[idx[d]][0], reverse=(d == 1))
                        grad[idx[d]][0] = dU
                        dzs.append(dz)
                    deltasOut = np.concatenate(dzs)
                else:
                    deltasOut = self._bptt(deltasOut, temporal[j], idx, grad, T)
            else:
                g = deltasOut * (hActs[i] > 0.0)
                if self.dropped(i):
                    g = g * float(threshold_scale(self.dropout)[1])
                if self.normed(i):
                    k = self.ln_index(i)
                    w_in, b_in = self.stack[i - 1]
                    xh, rstd = net_oracle.layer_norm(w_in.dot(self.map_input(hActs, i)) + b_in)
                    g, grad[k][0], grad[k][1] = net_oracle.layer_norm_backward(g, self.stack[k][0], xh, rstd)
                deltasOut = g
            deltasIn = deltasOut
        if self.reg > 0:
            for k in self.weight_indices():
                grad[k][0] += self.reg * self.stack[k][0]
        return cost, grad, skip
