"""lstm_oracle.py -- TEST INFRASTRUCTURE ONLY: NumPy restatement of a net whose temporal layers are LSTM cells.

The structure is stack_oracle.StackNet's: hidden layers 1..N, a block of numTemporal = k contiguous temporal layers
temporalLayer .. temporalLayer+k-1, the ReLU hidden layers and the linear output layer of the reference elsewhere, CTC
on top (brnn_oracle's, pinned to the reference's ctc_fast.pyx).  Each temporal layer is the LSTM cell of
include/ctcb200.h (cell = 1): its affine map has G = ndir*4H rows (forward direction first, gates i, f, g, o), each
recurrent matrix U is 4H x H, the layer output is h_f + h_b (uni-directional h_f).  Stack order and np.random draw
order are those of nnets.brnnet.NNet(cell='lstm').  Checked against torch.nn.LSTM and central finite differences in
tests/test_lstm_cpu.py.  Arrays are per utterance, [n][T] (the reference's layout)."""
import numpy as np

from oracle import brnn_oracle


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def lstm_direction(P, U, reverse):
    """One direction over one utterance: P = [4H][T] pre-activations, U = 4H x H.  Returns the activated gates
    [4H][T], c [H][T], h [H][T]."""
    H = U.shape[1]
    T = P.shape[1]
    gates = np.zeros_like(P)
    c = np.zeros((H, T), dtype=P.dtype)
    h = np.zeros((H, T), dtype=P.dtype)
    hp = np.zeros(H, dtype=P.dtype)
    cp = np.zeros(H, dtype=P.dtype)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        z = P[:, t] + U.dot(hp)
        i, f, g, o = _sig(z[:H]), _sig(z[H:2 * H]), np.tanh(z[2 * H:3 * H]), _sig(z[3 * H:])
        cp = f * cp + i * g
        hp = o * np.tanh(cp)
        gates[:, t] = np.concatenate([i, f, g, o])
        c[:, t], h[:, t] = cp, hp
    return gates, c, h


def lstm_direction_bptt(dh_in, gates, c, h, U, reverse):
    """BPTT of one direction given its activations: dh_in = [H][T] gradient w.r.t. the layer's output.  Returns dz
    [4H][T] and dU."""
    H = U.shape[1]
    T = dh_in.shape[1]
    dz = np.zeros_like(gates)
    dzn = np.zeros(4 * H, dtype=dh_in.dtype)
    dcn = np.zeros(H, dtype=dh_in.dtype)
    fn = np.zeros(H, dtype=dh_in.dtype)
    for t in (range(T) if reverse else range(T - 1, -1, -1)):
        i, f, g, o = gates[:H, t], gates[H:2 * H, t], gates[2 * H:3 * H, t], gates[3 * H:, t]
        dh = dh_in[:, t] + U.T.dot(dzn)
        tc = np.tanh(c[:, t])
        dc = dh * o * (1 - tc * tc) + dcn * fn
        tp = t + 1 if reverse else t - 1
        cprev = c[:, tp] if 0 <= tp < T else np.zeros(H, dtype=dh_in.dtype)
        dz[:, t] = np.concatenate([dc * g * i * (1 - i), dc * cprev * f * (1 - f), dc * i * (1 - g * g),
                                   dh * tc * o * (1 - o)])
        dzn, dcn, fn = dz[:, t], dc, f
    if reverse:
        dU = dz[:, :T - 1].dot(h[:, 1:].T)
    else:
        dU = dz[:, 1:].dot(h[:, :T - 1].T)
    return dz, dU


class LstmNet:
    def __init__(self, inputDim, outputDim, layerSize, numLayers, temporalLayer, numTemporal=1, reg=0.0,
                 unidirectional=False, dtype=np.float64, round_f32=True):
        assert 1 <= temporalLayer and temporalLayer + max(1, numTemporal) - 1 <= numLayers, "the block must fit"
        self.inputDim, self.outputDim, self.layerSize, self.numLayers = inputDim, outputDim, layerSize, numLayers
        self.temporalLayer, self.numTemporal = temporalLayer, max(1, numTemporal)
        self.reg, self.unidirectional, self.dtype, self.round_f32 = reg, unidirectional, dtype, round_f32
        self.ndir = 1 if unidirectional else 2
        self.G = self.ndir * 4 * layerSize
        self.regcost = 0.0

    def temporal(self, i):
        return self.temporalLayer <= i < self.temporalLayer + self.numTemporal

    def rec(self, j):
        base = self.numLayers + 1 + j * self.ndir
        return base, (None if self.unidirectional else base + 1)

    def shapes(self):
        """(rows, cols) of every tensor of the flat vector, in stack order (the library's table)."""
        H = self.layerSize
        sizes = [self.inputDim] + [H] * self.numLayers + [self.outputDim]
        out = []
        for i in range(1, self.numLayers + 2):
            m = self.G if self.temporal(i) else sizes[i]
            out += [(m, sizes[i - 1]), (m, 1)]
        for _ in range(self.numTemporal * self.ndir):
            out += [(4 * H, H), (1, 1)]
        return out

    def initParams(self):
        """nnets.brnnet.NNet(cell='lstm').initParams's draws: every matrix uniform in +-sqrt(6)/sqrt(rows+cols),
        biases 0, the maps first, then the recurrent matrices layer by layer; rounded to float32."""
        H = self.layerSize
        sizes = [self.inputDim] + [H] * self.numLayers + [self.outputDim]
        rows = [self.G if self.temporal(i) else sizes[i] for i in range(1, self.numLayers + 2)]
        scales = [np.sqrt(6) / np.sqrt(n + m) for n, m in zip(sizes[:-1], rows)]
        self.stack = [[np.random.rand(m, n) * 2 * s - s, np.zeros((m, 1))] for n, m, s in zip(sizes[:-1], rows, scales)]
        scale = np.sqrt(6) / np.sqrt(4 * H + H)
        for _ in range(self.numTemporal):
            for _ in range(self.ndir):
                self.stack.append([2 * scale * np.random.rand(4 * H, H) - scale, np.zeros((1, 1))])
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in self.stack]

    def _softmax(self, logits):
        z = logits - logits.max(axis=0)[None, :]
        e = np.exp(z)
        probs = e / e.sum(axis=0)[None, :]
        return probs.astype(np.float32) if self.round_f32 else probs

    def forward(self, data):
        """Returns (hActs [data, out_1 .. out_{N+1}], cells, probs); cells[j] = (gates [G][T], [c_f, c_b], [h_f, h_b])
        of temporal layer j (uni-directional: one entry per list)."""
        H = self.layerSize
        hActs = [np.asarray(data, dtype=self.dtype)]
        cells = []
        for i in range(1, self.numLayers + 2):
            w, b = self.stack[i - 1]
            x = w.dot(hActs[i - 1]) + b
            if self.temporal(i):
                gs, cs, hs = [], [], []
                for d, idx in enumerate(self.rec(i - self.temporalLayer)[:self.ndir]):
                    g, c, h = lstm_direction(x[d * 4 * H:(d + 1) * 4 * H], self.stack[idx][0], reverse=(d == 1))
                    gs.append(g)
                    cs.append(c)
                    hs.append(h)
                cells.append((np.concatenate(gs), cs, hs))
                x = sum(hs)
            elif i <= self.numLayers:
                x = np.maximum(x, 0.0)
            hActs.append(x)
        return hActs, cells, self._softmax(hActs[-1])

    def costAndGradGiven(self, data, labels, hActs, cells):
        """Back-propagation through GIVEN activations (out_1 .. out_{N+1} and each temporal layer's gates, c and h),
        e.g. the GPU's own."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(x, dtype=dt) for x in hActs]
        cells = [(np.asarray(g, dtype=dt), [np.asarray(c, dtype=dt) for c in cs], [np.asarray(h, dtype=dt) for h in hs])
                 for g, cs, hs in cells]
        return self.costAndGrad(data, labels, _given=(hActs, cells, self._softmax(hActs[-1])))

    def costAndGrad(self, data, labels, _given=None):
        hActs, cells, probs = self.forward(data) if _given is None else _given
        H = self.layerSize
        cost, deltas, skip = brnn_oracle._ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                                   np.asarray(labels, dtype=np.int32))
        grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        if self.reg > 0:
            self.regcost = sum((self.reg / 2.0) * float(np.sum(w.astype(np.float64) ** 2)) for w, _ in self.stack)
            cost = cost + self.regcost
        if skip:
            return cost, grad, skip
        deltasIn = (deltas.astype(np.float32) if self.round_f32 else deltas).astype(self.dtype)
        for i in range(self.numLayers, -1, -1):
            w = self.stack[i][0]
            grad[i][0] = deltasIn.dot(hActs[i].T)
            grad[i][1] = deltasIn.sum(axis=1)[:, None]
            if i == 0:
                break
            deltasOut = w.T.dot(deltasIn)
            if self.temporal(i):
                j = i - self.temporalLayer
                gates, cs, hs = cells[j]
                dzs = []
                for d, idx in enumerate(self.rec(j)[:self.ndir]):
                    dz, dU = lstm_direction_bptt(deltasOut, gates[d * 4 * H:(d + 1) * 4 * H], cs[d], hs[d],
                                                 self.stack[idx][0], reverse=(d == 1))
                    grad[idx][0] = dU
                    dzs.append(dz)
                deltasOut = np.concatenate(dzs)
            else:
                deltasOut = deltasOut * (hActs[i] > 0.0)
            deltasIn = deltasOut
        if self.reg > 0:
            for g, (w, _) in zip(grad, self.stack):
                g[0] += self.reg * w
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
        return np.array(costs), tot, np.array(skips)
