"""layernorm_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of a net whose ReLU hidden layers are
layer-normalised.

LayerNormNet is the float64 net of tests/dropout_oracle.py (DropoutNet over tests/stack_oracle.py: one or several
clipped-ReLU temporal layers, bi- or uni-directional, or none: the DNN; inverted dropout on the ReLU hidden layers) and,
with cell='lstm', the LSTM temporal layers of tests/lstm_oracle.py, with the normalisation of include/ctcb200.h
(layerNorm = 1) on every ReLU hidden layer that is not temporal:
    z = W x + b;  mu, var = mean, biased variance of z over the H units of a frame;  xh = (z - mu) / sqrt(var + 1e-5)
    X = relu(gamma * xh + beta)   (then dropout)
Stack order and np.random draw order are those of nnets.brnnet.NNet(layerNorm=True): the maps, the recurrent matrices,
then [gamma, beta] (H x 1 each, 1 and 0, no draw) of every normalised layer in ascending order.  The restatements it
builds on stay as they are.  Backward: g = dL/d(gamma xh + beta) = s * (W^T delta) * (X > 0) (s the dropout scale of a
dropped layer, else 1), dgamma = sum_t g xh, dbeta = sum_t g, dz = (g gamma - mean(g gamma) - xh mean(g gamma xh)) /
sqrt(var + 1e-5).  It is checked against torch.nn.functional.layer_norm and central finite differences in
tests/test_layernorm_cpu.py.  Arrays are per utterance, [n][T] (the reference's layout)."""
import numpy as np

from dropout_oracle import DropoutNet
from lstm_oracle import lstm_direction, lstm_direction_bptt
from oracle import brnn_oracle

EPS = 1e-5


def layer_norm(z, eps=EPS):
    """xh and rstd of the columns (frames) of z [H][T]: the normalisation over the units of each frame."""
    mu = z.mean(axis=0)
    var = ((z - mu) ** 2).mean(axis=0)
    rstd = 1.0 / np.sqrt(var + eps)
    return (z - mu) * rstd, rstd


def layer_norm_backward(g, gamma, xh, rstd):
    """dz, dgamma, dbeta of relu-free normalisation given g = dL/d(gamma xh + beta), [H][T]."""
    gh = g * gamma
    dz = rstd * (gh - gh.mean(axis=0) - xh * (gh * xh).mean(axis=0))
    return dz, (g * xh).sum(axis=1)[:, None], g.sum(axis=1)[:, None]


class LayerNormNet(DropoutNet):
    """DropoutNet (dropout=None: none) with cell 'relu' or 'lstm' and layer normalisation (layerNorm=False: none)."""

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal=1,
                 dropout=None, cell="relu", layerNorm=True, **kw):
        DropoutNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal,
                            dropout=dropout, **kw)
        self.cell, self.layerNorm = cell, layerNorm
        self.ndir = self.nrec

    def normed(self, i):
        return self.layerNorm and 1 <= i <= self.numLayers and not self.temporal(i)

    def normedLayers(self):
        return [i for i in range(1, self.numLayers + 1) if self.normed(i)]

    def ln_index(self, i):
        """Stack index of the [gamma, beta] pair of normalised layer i."""
        return self.numLayers + 1 + self.numTemporal * self.nrec + self.normedLayers().index(i)

    def map_rows(self, i):
        if self.cell == "lstm" and self.temporal(i):
            return self.ndir * 4 * self.layerSize
        return self.layerSize if i <= self.numLayers else self.outputDim

    def initParams(self):
        """nnets.brnnet.NNet.initParams's draws, rounded to float32."""
        H = self.layerSize
        sizes = [self.inputDim] + [H] * self.numLayers + [self.outputDim]
        rows = [self.map_rows(i) for i in range(1, self.numLayers + 2)]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(sizes[:-1], rows)]
        stack = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))] for n, m, s in zip(sizes[:-1], rows, scales)]
        rec_rows = 4 * H if self.cell == "lstm" else H
        scale = np.sqrt(6) / np.sqrt(rec_rows + H)
        for _ in range(self.numTemporal):
            for _ in range(self.nrec):
                stack.append([2 * scale * np.random.rand(rec_rows, H) - scale, np.zeros((1, 1))])
        stack += [[np.ones((H, 1)), np.zeros((H, 1))] for _ in self.normedLayers()]
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    def weight_indices(self):
        """Stack indices of the matrices L2 regularises: all but the [gamma, beta] pairs."""
        return range(self.numLayers + 1 + self.numTemporal * self.nrec)

    # ------------------------------------------------------------------ forward
    def forward(self, data):
        """Returns (hActs [data, X_1 .. X_{N+1}], temporal, probs); temporal[j] = (For, Back) of a clipped-ReLU layer
        (Back None uni-directional) or (gates, [c_f, c_b], [h_f, h_b]) of an LSTM layer."""
        H, T = self.layerSize, data.shape[1]
        hActs = [np.asarray(data, dtype=self.dtype)]
        temporal = []
        for i in range(1, self.numLayers + 2):
            w, b = self.stack[i - 1]
            z = w.dot(hActs[i - 1]) + b
            if self.temporal(i):
                idx = self.rec(i - self.temporalLayer)
                if self.cell == "lstm":
                    gs, cs, hs = [], [], []
                    for d in range(self.ndir):
                        g, c, h = lstm_direction(z[d * 4 * H:(d + 1) * 4 * H], self.stack[idx[d]][0], reverse=(d == 1))
                        gs.append(g)
                        cs.append(c)
                        hs.append(h)
                    temporal.append((np.concatenate(gs), cs, hs))
                    z = sum(hs)
                else:
                    For = self._sweep(z, self.stack[idx[0]][0], range(T), -1)
                    Back = None if self.unidirectional else self._sweep(z, self.stack[idx[1]][0],
                                                                       range(T - 1, -1, -1), 1)
                    temporal.append((For, Back))
                    z = For if Back is None else For + Back
            elif i <= self.numLayers:
                if self.normed(i):
                    gamma, beta = self.stack[self.ln_index(i)]
                    z = gamma * layer_norm(z)[0] + beta
                z = np.maximum(z, 0.0)
                if self.dropped(i):
                    z = self.dropout.apply(z, i)
            hActs.append(z)
        return hActs, temporal, self._softmax(hActs[-1])

    # ------------------------------------------------------------------ backward
    def costAndGradGiven(self, data, labels, hActs, temporal):
        """Back-propagation through GIVEN activations (X_1 .. X_{N+1} and each temporal layer's own, e.g. the GPU's):
        the ReLU and dropout masks are X_i > 0, and each normalised layer's xh and rstd are recomputed in float64
        from the given input of its map."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(x, dtype=dt) for x in hActs]
        cvt = lambda x: None if x is None else (np.asarray(x, dtype=dt) if not isinstance(x, list)  # noqa: E731
                                                 else [np.asarray(y, dtype=dt) for y in x])
        temporal = [tuple(cvt(x) for x in t) for t in temporal]
        return self.costAndGrad(data, labels, _given=(hActs, temporal, self._softmax(hActs[-1])))

    def costAndGrad(self, data, labels, _given=None):
        hActs, temporal, probs = self.forward(data) if _given is None else _given
        H, T, dt = self.layerSize, data.shape[1], self.dtype
        cost, deltas, skip = brnn_oracle._ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                                   np.asarray(labels, dtype=np.int32))
        grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        if self.reg > 0:
            self.regcost = sum((self.reg / 2.0) * float(np.sum(self.stack[k][0].astype(np.float64) ** 2))
                               for k in self.weight_indices())
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
                idx = self.rec(j)
                if self.cell == "lstm":
                    gates, cs, hs = temporal[j]
                    dzs = []
                    for d in range(self.ndir):
                        dz, dU = lstm_direction_bptt(deltasOut, gates[d * 4 * H:(d + 1) * 4 * H], cs[d], hs[d],
                                                     self.stack[idx[d]][0], reverse=(d == 1))
                        grad[idx[d]][0] = dU
                        dzs.append(dz)
                    deltasOut = np.concatenate(dzs)
                else:
                    deltasOut = self._bptt(deltasOut, temporal[j], idx, grad, T)
            else:
                g = deltasOut * (hActs[i] > 0.0)
                if self.dropped(i):
                    g = g * float(self.dropout.scale)
                if self.normed(i):
                    k = self.ln_index(i)
                    w_in, b_in = self.stack[i - 1]
                    xh, rstd = layer_norm(w_in.dot(hActs[i - 1]) + b_in)
                    g, grad[k][0], grad[k][1] = layer_norm_backward(g, self.stack[k][0], xh, rstd)
                deltasOut = g
            deltasIn = deltasOut
        if self.reg > 0:
            for k in self.weight_indices():
                grad[k][0] += self.reg * self.stack[k][0]
        self.grad = grad
        return cost, grad, skip

    def _bptt(self, pre, temporal, idx, grad, T):
        """The clipped-ReLU BPTT of stack_oracle.StackNet (brnnet.py:207-233) for one temporal layer."""
        For, Back = temporal
        dt = self.dtype
        mF = ((For > 0.0) & (For < self.maxAct)).astype(dt)
        wtf = self.stack[idx[0]][0]
        dFor = pre.copy()
        dFor[:, T - 1] *= mF[:, T - 1]
        for t in range(T - 1, 0, -1):
            dFor[:, t - 1] += wtf.T.dot(dFor[:, t])
            dFor[:, t - 1] *= mF[:, t - 1]
        grad[idx[0]][0] = dFor[:, 1:T].dot(For[:, 0:T - 1].T)
        if Back is None:
            return dFor
        mB = ((Back > 0.0) & (Back < self.maxAct)).astype(dt)
        wtb = self.stack[idx[1]][0]
        dBack = pre.copy()
        dBack[:, 0] *= mB[:, 0]
        for t in range(1, T):
            dBack[:, t] += wtb.T.dot(dBack[:, t - 1])
            dBack[:, t] *= mB[:, t]
        grad[idx[1]][0] = dBack[:, 0:T - 1].dot(Back[:, 1:T].T)
        return dFor + dBack

    def costAndGradBatch(self, datas, labelss, utts=None):
        """Per-utterance gradients summed (a skipped utterance adds nothing), the L2 term added once to the weight
        matrices; utterance u draws the dropout mask of minibatch index utts[u] (default u)."""
        reg, self.reg = self.reg, 0.0
        tot = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        costs, skips = [], []
        for u, (d, l) in enumerate(zip(datas, labelss)):
            if self.dropout is not None:
                self.dropout.g = u if utts is None else utts[u]
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
            for k in self.weight_indices():
                w = self.stack[k][0]
                self.regcost += (reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                tot[k][0] += reg * w
        self.grad = tot
        return np.array(costs), self.grad, np.array(skips)
