"""subsample_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of a net that runs its upper layers at a reduced
frame rate (include/ctcb200.h: subsample).

SubsampleNet is the float64 net of tests/layernorm_oracle.py (LayerNormNet: clipped-ReLU or LSTM temporal layers, one
or a stack, bi- or uni-directional, or none; dropout and layer normalisation of the ReLU hidden layers) in which affine
map L = subsampleLayer reads k consecutive frames of the layer below it, concatenated:
    S[:, t'] = [x_{k t'}; x_{k t' + 1}; ...; x_{k t' + k - 1}]     (rows m n .. m n + n - 1 hold sub-frame m)
with x_t = 0 for t >= T, so map L and everything above it (temporal layers, softmax, CTC) run on T' = ceil(T / k)
frames.  Dropout draws with the frame index of the layer's own rate.  W_L is rows x k n, drawn at fan-in k n in the
draw order of nnets.brnnet.NNet.initParams.  Backward: dW_L = delta_L S^T and the delta of layer L - 1 is W_L^T delta_L
unstacked to T frames (sub-frames beyond T dropped), then masked as without subsampling.  Arrays are per utterance,
[n][T] (the reference's layout).  It is checked against torch autograd and central differences in
tests/test_subsample_cpu.py."""
import numpy as np

from layernorm_oracle import LayerNormNet, layer_norm, layer_norm_backward
from lstm_oracle import lstm_direction, lstm_direction_bptt
from oracle import brnn_oracle


def frames(T, k):
    return -(-T // k) if k > 1 else T


def stack_frames(x, k):
    """[n][T] -> [k n][ceil(T / k)], zero beyond T."""
    n, T = x.shape
    Tp = frames(T, k)
    pad = np.zeros((n, Tp * k), dtype=x.dtype)
    pad[:, :T] = x
    return pad.T.reshape(Tp, k * n).T.copy()


def unstack_frames(d, k, T):
    """[k n][T'] -> [n][T]: the inverse of stack_frames on the first T frames."""
    kn, Tp = d.shape
    return d.T.reshape(Tp * k, kn // k)[:T].T.copy()


class SubsampleNet(LayerNormNet):
    """LayerNormNet (layerNorm=False: none) with subsample=k at map subsampleLayer=L (k <= 1: off)."""

    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal=1,
                 subsample=2, subsampleLayer=1, layerNorm=False, **kw):
        LayerNormNet.__init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer, numTemporal,
                              layerNorm=layerNorm, **kw)
        self.k, self.L = (subsample, subsampleLayer) if subsample > 1 else (1, 0)

    def stacked(self, i):
        return self.k > 1 and i == self.L

    def map_cols(self, i):
        n = self.inputDim if i == 1 else self.layerSize
        return self.k * n if self.stacked(i) else n

    def initParams(self):
        H = self.layerSize
        cols = [self.map_cols(i) for i in range(1, self.numLayers + 2)]
        rows = [self.map_rows(i) for i in range(1, self.numLayers + 2)]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(cols, rows)]
        stack = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))] for n, m, s in zip(cols, rows, scales)]
        rec_rows = 4 * H if self.cell == "lstm" else H
        scale = np.sqrt(6) / np.sqrt(rec_rows + H)
        for _ in range(self.numTemporal):
            for _ in range(self.nrec):
                stack.append([2 * scale * np.random.rand(rec_rows, H) - scale, np.zeros((1, 1))])
        stack += [[np.ones((H, 1)), np.zeros((H, 1))] for _ in self.normedLayers()]
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    def map_input(self, hActs, i):
        """What affine map i reads: X_{i-1}, or S stacked from it at map L."""
        return stack_frames(hActs[i - 1], self.k) if self.stacked(i) else hActs[i - 1]

    # ------------------------------------------------------------------ forward
    def forward(self, data):
        """(hActs [data, X_1 .. X_{N+1}], temporal, probs) as LayerNormNet's, X_i on T' frames from map L up."""
        H = self.layerSize
        hActs = [np.asarray(data, dtype=self.dtype)]
        temporal = []
        for i in range(1, self.numLayers + 2):
            w, b = self.stack[i - 1]
            z = w.dot(self.map_input(hActs, i)) + b
            T = z.shape[1]
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
    def costAndGrad(self, data, labels, _given=None):
        hActs, temporal, probs = self.forward(data) if _given is None else _given
        H, dt = self.layerSize, self.dtype
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
            grad[i][0] = deltasIn.dot(self.map_input(hActs, i + 1).T)
            grad[i][1] = deltasIn.sum(axis=1)[:, None]
            if i == 0:
                break
            deltasOut = w.T.dot(deltasIn)
            if self.stacked(i + 1):
                deltasOut = unstack_frames(deltasOut, self.k, hActs[i].shape[1])
            T = deltasOut.shape[1]
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
                    xh, rstd = layer_norm(w_in.dot(self.map_input(hActs, i)) + b_in)
                    g, grad[k][0], grad[k][1] = layer_norm_backward(g, self.stack[k][0], xh, rstd)
                deltasOut = g
            deltasIn = deltasOut
        if self.reg > 0:
            for k in self.weight_indices():
                grad[k][0] += self.reg * self.stack[k][0]
        self.grad = grad
        return cost, grad, skip
