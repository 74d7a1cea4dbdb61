"""dropout_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of libctcb200's inverted dropout.

The mask of include/ctcb200.h (ctcb_brnn_set_dropout) in NumPy -- Philox4x32-10, the threshold and the scale -- and
DropoutNet, the float64 net of tests/stack_oracle.py (one or several temporal layers, bi- or uni-directional, or none:
the DNN) with that dropout on the outputs of its ReLU hidden layers.  The restatements it builds on stay as they are.

Backward pass: a dropped layer i has X_i = s * m * relu(z_i), so dL/dz_i = s * (W_{i+1}^T delta_{i+1}) * (X_i > 0).
StackNet's back-propagation computes the same recursion without the factors s; the recursion (BPTT included) is linear
in the deltas once the masks are fixed, so its delta of layer j is the true one divided by s^(number of dropped layers
at or above j), and DropoutNet multiplies each gradient tensor by that power.  The masks come from the activations,
given or computed, as StackNet's do."""
import numpy as np

from stack_oracle import StackNet

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11; curand_Philox4x32_10) of counters ctr (..., 4) under key (k0, k1);
    returns (..., 4) uint32."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for rnd in range(10):
        if rnd:
            k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0)) & _U32, p1 & _U32,
             ((p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1)) & _U32, p0 & _U32]
    return np.stack(c, axis=-1).astype(np.uint32)


def threshold_scale(p):
    """(thr, s) for the float32 p the library is given: keep iff draw >= thr, a kept x becomes x * s."""
    pd = float(np.float32(p))
    return int(np.floor(pd * 4294967296.0)), np.float32(1.0 / (1.0 - pd))


def draws(seed, step, layer, g, T, H):
    """Philox outputs of units 0..H-1 of frames 0..T-1 of minibatch utterance g in hidden layer `layer` at `step`:
    uint32 (T, H), the device's time-major order."""
    Q = (H + 3) // 4
    t, q = np.meshgrid(np.arange(T, dtype=np.uint64), np.arange(Q, dtype=np.uint64), indexing="ij")
    ctr = np.stack([np.full_like(t, int(step) & 0xFFFFFFFF), np.full_like(t, int(g) & 0xFFFFFFFF), t,
                    np.uint64(int(layer) << 24) | q], axis=-1)
    r = philox4x32_10(ctr, (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF))
    return r.reshape(T, 4 * Q)[:, :H]


def keep_mask(p, seed, step, layer, g, T, H):
    """Boolean (T, H) keep mask of one utterance's hidden layer."""
    return draws(seed, step, layer, g, T, H) >= np.uint32(threshold_scale(p)[0])


class Dropout(object):
    """What a DropoutNet drops: p, seed, the step whose mask is drawn and the minibatch index g of the utterance being
    computed (costAndGradBatch sets it per utterance)."""

    def __init__(self, p, seed=33, step=0, g=0):
        self.p, self.seed, self.step, self.g = p, seed, step, g
        self.scale = threshold_scale(p)[1]

    def apply(self, h, layer):
        """An (H, T) activation times mask * s, in h's dtype (s is the float32 scale, widened exactly)."""
        keep = keep_mask(self.p, self.seed, self.step, layer, self.g, h.shape[1], h.shape[0]).T
        return np.where(keep, h * h.dtype.type(self.scale), h.dtype.type(0))


class DropoutNet(StackNet):
    """StackNet with dropout (None: StackNet itself).  temporalLayer <= 0 is the DNN of nnets/nnet.py."""

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal=1,
                 dropout=None, **kw):
        dnn = temporalLayer <= 0
        StackNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, 1 if dnn else temporalLayer,
                          numTemporal, **kw)
        if dnn:
            self.temporalLayer, self.numTemporal = 0, 0
        self.dropout = dropout

    def dropped(self, i):
        return self.dropout is not None and 1 <= i <= self.numLayers and not self.temporal(i)

    def forward(self, data):
        T = data.shape[1]
        hActs = [np.asarray(data, dtype=self.dtype)]
        Fors, Backs = [], []
        for i in range(1, self.numLayers + 2):
            w, b = self.stack[i - 1]
            h = w.dot(hActs[i - 1]) + b
            if self.temporal(i):
                f_idx, b_idx = self.rec(i - self.temporalLayer)
                For = self._sweep(h, self.stack[f_idx][0], range(T), -1)
                Fors.append(For)
                if self.unidirectional:
                    h = For
                    Backs.append(None)
                else:
                    Back = self._sweep(h, self.stack[b_idx][0], range(T - 1, -1, -1), 1)
                    Backs.append(Back)
                    h = For + Back
            elif i <= self.numLayers:
                h = np.maximum(h, 0.0)
                if self.dropped(i):
                    h = self.dropout.apply(h, i)
            hActs.append(h)
        return hActs, Fors, (None if self.unidirectional else Backs), self._softmax(hActs[-1])

    def _sweep(self, pre, wt, order, prev):
        """Clipped-ReLU recurrence over the frames in `order`, each reading the frame at offset `prev`."""
        out = pre.copy()
        for n, t in enumerate(order):
            if n:
                out[:, t] = out[:, t] + wt.dot(out[:, t + prev])
            out[:, t] = np.clip(out[:, t], 0.0, self.maxAct)
        return out

    def costAndGrad(self, data, labels, _given=None):
        given = self.forward(data) if _given is None else _given
        cost, grad, skip = StackNet.costAndGrad(self, data, labels, _given=given)
        if self.dropout is None or skip:
            return cost, grad, skip
        s = float(self.dropout.scale)
        above = lambda j: sum(self.dropped(i) for i in range(j, self.numLayers + 1))    # noqa: E731
        for idx, (gw, gb) in enumerate(grad):
            # map idx + 1 (its delta is that of layer idx + 1), or a recurrent matrix of temporal layer i
            j = idx + 1 if idx <= self.numLayers else self.temporalLayer + (idx - self.numLayers - 1) // self.nrec
            f = s ** above(j)
            w = self.stack[idx][0]
            gw[...] = f * (gw - self.reg * w) + self.reg * w
            gb[...] = f * gb
        return cost, grad, skip

    def costAndGradBatch(self, datas, labelss, utts=None):
        """StackNet.costAndGradBatch with utterance u drawing the mask of minibatch index utts[u] (default u)."""
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
            for (w, _), (tw, _) in zip(self.stack, tot):
                self.regcost += (reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2))
                tw += reg * w
        self.grad = tot
        return np.array(costs), self.grad, np.array(skips)
