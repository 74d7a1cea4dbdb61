"""net_oracle.py -- TEST INFRASTRUCTURE ONLY: one NumPy float64 restatement of every net nnets.brnnet.NNet builds.

The one-temporal-layer restatement (oracle/brnn_oracle.py) is pinned to the reference's own rnnetcpu.py and stays as it
is; with every feature off, Net computes what it computes.  Net takes NNet's keyword arguments with their names,
defaults and validity rules, so a test builds the device net and its oracle from one dict:
  * hidden layers 1..N and the linear output map N+1; a block of numTemporal = k contiguous temporal layers
    temporalLayer .. temporalLayer+k-1 (temporalLayer <= 0, or at or above hi: none, the DNN of nnets/nnet.py; hi =
    N + 1 with allowTopTemporal, else N), bi- or uni-directional; the ReLU hidden layers elsewhere.
  * cell='relu': the clipped-ReLU recurrence of brnnet.py:143-153 / rnnet.py:112-116, back-propagated with the BPTT of
    brnnet.py:207-233 / rnnet.py:162-177.  cell='lstm': the LSTM cell of include/ctcb200.h (cell = 1), whose map has
    ndir*4H rows (forward direction first, gates i, f, g, o) and whose recurrent matrices U are 4H x H; the layer
    output is h_f + h_b (uni-directional h_f).
  * layerNorm: every ReLU hidden layer is z = W x + b; xh = (z - mean) / sqrt(biased var + 1e-5) over the H units of a
    frame; X = relu(gamma xh + beta).  Backward: g = dL/d(gamma xh + beta), dgamma = sum_t g xh, dbeta = sum_t g,
    dz = (g gamma - mean(g gamma) - xh mean(g gamma xh)) / sqrt(var + 1e-5).
  * dropout = p: inverted dropout on the outputs of the ReLU hidden layers with the Philox4x32-10 mask of
    ctcb_brnn_set_dropout, drawn for step dropoutStep and minibatch utterance utt; a dropped layer has
    X_i = s * m * relu(z_i), so dL/dz_i = s * (W_{i+1}^T delta_{i+1}) * (X_i > 0).
  * subsample = k at map L = subsampleLayer: map L reads k consecutive frames of the layer below it, concatenated,
    S[:, t'] = [x_{k t'}; ..; x_{k t' + k - 1}] with x_t = 0 for t >= T, so map L and everything above it run on
    T' = ceil(T / k) frames.  dW_L = delta_L S^T; the delta of layer L - 1 is W_L^T delta_L unstacked to T frames.
Stack order and np.random draw order are those of NNet.initParams: the maps, the recurrent matrices layer by layer
([Wtf_j, dummy] [Wtb_j, dummy]), then [gamma, beta] of every normalised layer.  L2 adds reg * W to every weight matrix,
recurrent ones included, not to the [gamma, beta] pairs.  The CTC half is brnn_oracle's (pinned to the reference's
ctc_fast.pyx).  Arrays are per utterance, [n][T] (the reference's layout).  Checked against torch and central finite
differences in tests/test_net_oracle_cpu.py."""
import numpy as np

from oracle import brnn_oracle

EPS = 1e-5
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_U32 = np.uint64(0xFFFFFFFF)


# ------------------------------------------------------------------------------------------------ dropout mask
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


# ------------------------------------------------------------------------------------------------ LSTM cell
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


# ------------------------------------------------------------------------------------------------ layer norm
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


# ------------------------------------------------------------------------------------------------ subsampling
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


# ------------------------------------------------------------------------------------------------ the net
class Net:
    def __init__(self, inputDim, outputDim, layerSize, numLayers, maxBatch, temporalLayer=-1, reg=0.0,
                 unidirectional=False, numTemporal=1, allowTopTemporal=False, cell="relu", layerNorm=False,
                 subsample=1, subsampleLayer=1, dropout=0.0, dropoutSeed=33, dtype=np.float64, round_f32=True):
        hi = numLayers + 1 if allowTopTemporal else numLayers
        if numTemporal < 0:
            raise ValueError("numTemporal=%d must be >= 0" % numTemporal)
        if numTemporal > 1 and (temporalLayer <= 0 or temporalLayer + numTemporal - 1 >= hi):
            raise ValueError("numTemporal=%d from temporalLayer=%d does not fit" % (numTemporal, temporalLayer))
        if cell not in ("relu", "lstm"):
            raise ValueError("cell=%r" % (cell,))
        if not 0.0 <= dropout < 1.0:
            raise ValueError("dropout=%r must be in [0, 1)" % (dropout,))
        self.inputDim, self.outputDim, self.layerSize, self.numLayers = inputDim, outputDim, layerSize, numLayers
        self.maxBatch, self.reg, self.dtype, self.round_f32 = maxBatch, reg, dtype, round_f32
        self.temporalLayer = temporalLayer if 0 < temporalLayer < hi else -1
        self.numTemporal = max(1, numTemporal) if self.temporalLayer > 0 else 0
        self.unidirectional, self.cell, self.layerNorm = bool(unidirectional), cell, bool(layerNorm)
        self.nrec = 1 if self.unidirectional else 2
        self.k, self.L = (int(subsample), int(subsampleLayer)) if subsample > 1 else (1, 0)
        self.dropout, self.dropoutSeed = float(dropout), int(dropoutSeed)
        self.dropoutStep, self.utt = 0, 0       # the mask's step and the minibatch index of the utterance computed
        self.maxAct = 20.0
        self.regcost = 0.0

    # ------------------------------------------------------------------ structure
    def temporal(self, i):
        return self.numTemporal > 0 and self.temporalLayer <= i < self.temporalLayer + self.numTemporal

    def rec(self, j):
        """Stack indices of the recurrent matrices of temporal layer j (0-based within the block)."""
        base = self.numLayers + 1 + j * self.nrec
        return base, (None if self.unidirectional else base + 1)

    def dropped(self, i):
        return self.dropout > 0.0 and 1 <= i <= self.numLayers and not self.temporal(i)

    def normed(self, i):
        return self.layerNorm and 1 <= i <= self.numLayers and not self.temporal(i)

    def normedLayers(self):
        return [i for i in range(1, self.numLayers + 1) if self.normed(i)]

    def ln_index(self, i):
        """Stack index of the [gamma, beta] pair of normalised layer i."""
        return self.numLayers + 1 + self.numTemporal * self.nrec + self.normedLayers().index(i)

    def weight_indices(self):
        """Stack indices of the matrices L2 regularises: all but the [gamma, beta] pairs."""
        return range(self.numLayers + 1 + self.numTemporal * self.nrec)

    def stacked(self, i):
        return self.k > 1 and i == self.L

    def shapes(self):
        """(rows, cols) of every tensor of the flat vector, in stack order (the library's table)."""
        H = self.layerSize
        out = []
        for i in range(1, self.numLayers + 2):
            m = self.layerSize if i <= self.numLayers else self.outputDim
            if self.cell == "lstm" and self.temporal(i):
                m = self.nrec * 4 * H
            n = self.inputDim if i == 1 else H
            out += [(m, self.k * n if self.stacked(i) else n), (m, 1)]
        out += [(4 * H if self.cell == "lstm" else H, H), (1, 1)] * (self.numTemporal * self.nrec)
        return out + [(H, 1), (H, 1)] * len(self.normedLayers())

    def initParams(self):
        """NNet.initParams's draws, rounded to float32: every matrix uniform in +-sqrt(6)/sqrt(rows+cols), biases 0,
        gamma 1 and beta 0 without a draw."""
        shapes = self.shapes()
        nw = len(self.weight_indices())
        stack = []
        for t, ((m, n), bshape) in enumerate(zip(shapes[0::2], shapes[1::2])):
            if t <= self.numLayers:
                s = np.sqrt(6) / np.sqrt(n + m)
                stack.append([np.random.rand(m, n) * 2 * s - s, np.zeros(bshape)])
            elif t < nw:
                scale = np.sqrt(6) / np.sqrt(m + n)
                stack.append([2 * scale * np.random.rand(m, n) - scale, np.zeros(bshape)])
            else:
                stack.append([np.ones((m, n)), np.zeros(bshape)])
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    # ------------------------------------------------------------------ forward
    def drop(self, h, layer):
        """An (H, T) activation of hidden layer `layer` times mask * s, in h's dtype (s is the float32 scale, widened
        exactly)."""
        keep = keep_mask(self.dropout, self.dropoutSeed, self.dropoutStep, layer, self.utt, h.shape[1], h.shape[0]).T
        return np.where(keep, h * h.dtype.type(threshold_scale(self.dropout)[1]), h.dtype.type(0))

    def map_input(self, hActs, i):
        """What affine map i reads: X_{i-1}, or S stacked from it at map L."""
        return stack_frames(hActs[i - 1], self.k) if self.stacked(i) else hActs[i - 1]

    def _softmax(self, logits):
        z = logits - logits.max(axis=0)[None, :]
        e = np.exp(z)
        probs = e / e.sum(axis=0)[None, :]
        return probs.astype(np.float32) if self.round_f32 else probs

    def _sweep(self, pre, wt, order, prev):
        """Clipped-ReLU recurrence over the frames in `order`, each reading the frame at offset `prev`."""
        out = pre.copy()
        for n, t in enumerate(order):
            if n:
                out[:, t] = out[:, t] + wt.dot(out[:, t + prev])
            out[:, t] = np.clip(out[:, t], 0.0, self.maxAct)
        return out

    def forward(self, data):
        """Returns (hActs [data, X_1 .. X_{N+1}], temporal, probs), X_i on T' frames from map L up; temporal[j] =
        (For, Back) of a clipped-ReLU layer (Back None uni-directional) or (gates, [c_f, c_b], [h_f, h_b]) of an LSTM
        layer."""
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
                    for d in range(self.nrec):
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
                    z = self.drop(z, i)
            hActs.append(z)
        return hActs, temporal, self._softmax(hActs[-1])

    # ------------------------------------------------------------------ backward
    def costAndGradGiven(self, data, labels, hActs, temporal):
        """Back-propagation through GIVEN activations (X_1 .. X_{N+1} and each temporal layer's own, as `forward`
        returns them, e.g. the GPU's): the ReLU, clip and dropout masks are the given arrays' (X_i > 0), and each
        normalised layer's xh and rstd are recomputed in float64 from the given input of its map."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(x, dtype=dt) for x in hActs]
        cvt = lambda x: None if x is None else (np.asarray(x, dtype=dt) if not isinstance(x, list)  # noqa: E731
                                                 else [np.asarray(y, dtype=dt) for y in x])
        temporal = [tuple(cvt(x) for x in t) for t in temporal]
        return self.costAndGrad(data, labels, _given=(hActs, temporal, self._softmax(hActs[-1])))

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
                    for d in range(self.nrec):
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
                    g = g * float(threshold_scale(self.dropout)[1])
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

    def _bptt(self, pre, temporal, idx, grad, T):
        """The clipped-ReLU BPTT (brnnet.py:207-233, rnnet.py:162-177) of one temporal layer."""
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
            self.utt = u if utts is None else utts[u]
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
