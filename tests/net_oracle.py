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
  * peephole (include/ctcb200.h: peephole = 1): per LSTM direction P = [p_i; p_f; p_o] (3 x H), i = sigmoid(z_i +
    p_i c_prev), f = sigmoid(z_f + p_f c_prev), o = sigmoid(z_o + p_o c_t), c_prev = c_{t-1} (c_{t+1} backward in time)
    and 0 before the first frame.  dp_i = sum dz_i c_prev, dp_f = sum dz_f c_prev, dp_o = sum dz_o c.
  * zoneoutCell = z_c, zoneoutHidden = z_h (zoneout = 1): unit j of frame t (at the layer's rate) of minibatch
    utterance g in direction d of temporal layer i at step s draws (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod
    2^32, g mod 2^32, t, (i << 24) | (d << 23) | j), key = (seed mod 2^32, seed >> 32)); lambda_c = 1 iff r0 < floor(z_c
    2^32), lambda_h = 1 iff r1 < floor(z_h 2^32).  With `expectation` set (forward-only calls) lambda = float32(z).
    c~ = f c_prev + i g;  c = lc c_prev + (1 - lc) c~;  h = lh h_prev + (1 - lh) o tanh(c)  (i, f see the zoned
    c_prev, o the zoned c).  BPTT ("next" = the step after t in the direction's order):
        dh = delta + U^T dz_next + lh_next dh_next;  dh~ = (1 - lh) dh;  dz_o = dh~ tanh(c) o(1-o)
        dc = dh~ o (1 - tanh^2 c) + p_o dz_o + (lc_next + (1 - lc_next) f_next) dc_next + p_i dz_i,next + p_f dz_f,next
        dc~ = (1 - lc) dc;  dz_i = dc~ g i(1-i);  dz_f = dc~ c_prev f(1-f);  dz_g = dc~ i(1-g^2)
    There is one LSTM cell: without peepholes P = 0, without zoneout lambda = 0, and every extra term is then an exact
    + 0 x or 1 x in float64, so such a net computes the plain cell's numbers bit for bit.
  * interLayer = m, interWeight = lambda: hidden layer m's output X_m goes through the output map, A = W_{N+1} X_m +
    b_{N+1} on layer m's own frames, and the objective is nll_main + lambda nll_aux (lambda the float32 the library is
    given).  The intermediate term's gradient is that of the HEAD NET (head()): hidden layers 1..m with the output map
    on top, over the very arrays of this net's stack, so it computes X_m as this net does, bit for bit.  Each CTC skips
    on its own: costAndGrad returns (main cost, gradient of the objective, main skip) and leaves the intermediate nll
    and skip in interCost / interSkip.
  * selfCondition: map m + 1 (and the frame stacking, when it starts there) reads X'_m = X_m + W_c P + b_c, P =
    softmax(A) per frame.  Backward at layer m: D'_m = W_{m+1}^T delta_{m+1} (unstacked), dP = W_c^T D'_m, dA = P (dP -
    sum_k P_k dP_k), dW_c = D'_m P^T, db_c = sum_t D'_m, dW_{N+1} += dA X_m^T, db_{N+1} += sum_t dA, and
    D'_m + W_{N+1}^T dA is the delta that layer m's mask, normalisation or BPTT then reads.
Stack order and np.random draw order are those of NNet.initParams: the maps, the recurrent matrices layer by layer
([Wtf_j, dummy] [Wtb_j, dummy]), then [gamma, beta] of every normalised layer, then [P, dummy] of every direction of
every LSTM layer with peepholes, then [W_c (H x K), b_c (H x 1)]; P, W_c and b_c are 0 and take no draw.  L2 adds
reg * W to every weight matrix, recurrent ones included, not to the [gamma, beta], [P, dummy] or [W_c, b_c] pairs.  The
CTC half is brnn_oracle's (pinned to the reference's ctc_fast.pyx).  Arrays are per utterance, [n][T] (the reference's
layout).
Checked against torch and central finite differences in tests/test_net_oracle_cpu.py and the feature CPU tests."""
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


# ------------------------------------------------------------------------------------------------ zoneout masks
def zoneout_threshold(z):
    """floor(z 2^32) of the float32 z the library is given, in float64."""
    return int(np.floor(float(np.float32(z)) * 4294967296.0))


def zoneout_draws(seed, step, layer, d, g, T, H):
    """Philox outputs (T, H, 4) uint32 of units 0..H-1 of frames 0..T-1 of minibatch utterance g, direction d of
    temporal layer `layer`, at `step`."""
    t, j = np.meshgrid(np.arange(T, dtype=np.uint64), np.arange(H, dtype=np.uint64), indexing="ij")
    ctr = np.stack([np.full_like(t, int(step) & 0xFFFFFFFF), np.full_like(t, int(g) & 0xFFFFFFFF), t,
                    np.uint64((int(layer) << 24) | (int(d) << 23)) | j], axis=-1)
    return philox4x32_10(ctr, (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF))


def zoneout_masks(zc, zh, seed, step, layer, d, g, T, H):
    """Boolean (T, H) lambda_c and lambda_h of one direction of one utterance (True: keep the previous value)."""
    r = zoneout_draws(seed, step, layer, d, g, T, H)
    return r[..., 0] < np.uint32(zoneout_threshold(zc)), r[..., 1] < np.uint32(zoneout_threshold(zh))


# ------------------------------------------------------------------------------------------------ LSTM cell
def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def lstm_direction(P, U, reverse, peep, lc, lh):
    """One direction over one utterance: P = [4H][T] pre-activations, U = 4H x H, peep its 3 x H [p_i; p_f; p_o], lc /
    lh [H][T] its zoneout lambdas.  Returns the activated gates [4H][T] (o after its peephole), c [H][T] and h [H][T]
    (the zoned c and h)."""
    H = U.shape[1]
    T = P.shape[1]
    gates = np.zeros_like(P)
    c = np.zeros((H, T), dtype=P.dtype)
    h = np.zeros((H, T), dtype=P.dtype)
    hp = np.zeros(H, dtype=P.dtype)
    cp = np.zeros(H, dtype=P.dtype)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        z = P[:, t] + U.dot(hp)
        i, f, g = _sig(z[:H] + peep[0] * cp), _sig(z[H:2 * H] + peep[1] * cp), np.tanh(z[2 * H:3 * H])
        cp = lc[:, t] * cp + (1 - lc[:, t]) * (f * cp + i * g)
        o = _sig(z[3 * H:] + peep[2] * cp)
        hp = lh[:, t] * hp + (1 - lh[:, t]) * (o * np.tanh(cp))
        gates[:, t] = np.concatenate([i, f, g, o])
        c[:, t], h[:, t] = cp, hp
    return gates, c, h


def lstm_direction_bptt(dh_in, gates, c, h, U, reverse, peep, lc, lh):
    """BPTT of one direction given its activations: dh_in = [H][T] gradient w.r.t. the layer's output.  Returns dz
    [4H][T], dU and dP (3 x H)."""
    H = U.shape[1]
    T = dh_in.shape[1]
    dt = dh_in.dtype
    dz = np.zeros_like(gates)
    dzn, dcn, fn = np.zeros(4 * H, dtype=dt), np.zeros(H, dtype=dt), np.zeros(H, dtype=dt)
    dhn, lcn, lhn = np.zeros(H, dtype=dt), np.zeros(H, dtype=dt), np.zeros(H, dtype=dt)
    dP = np.zeros((3, H), dtype=dt)
    for t in (range(T) if reverse else range(T - 1, -1, -1)):
        i, f, g, o = gates[:H, t], gates[H:2 * H, t], gates[2 * H:3 * H, t], gates[3 * H:, t]
        dh = dh_in[:, t] + U.T.dot(dzn) + lhn * dhn
        dht = (1 - lh[:, t]) * dh
        tc = np.tanh(c[:, t])
        tp = t + 1 if reverse else t - 1
        cprev = c[:, tp] if 0 <= tp < T else np.zeros(H, dtype=dt)
        dzo = dht * tc * o * (1 - o)
        carry = (lcn + (1 - lcn) * fn) * dcn
        dc = dht * o * (1 - tc * tc) + peep[2] * dzo + carry + peep[0] * dzn[:H] + peep[1] * dzn[H:2 * H]
        dcc = (1 - lc[:, t]) * dc
        dz[:, t] = np.concatenate([dcc * g * i * (1 - i), dcc * cprev * f * (1 - f), dcc * i * (1 - g * g), dzo])
        dP[0] += dz[:H, t] * cprev
        dP[1] += dz[H:2 * H, t] * cprev
        dP[2] += dzo * c[:, t]
        dzn, dcn, fn, dhn, lcn, lhn = dz[:, t], dc, f, dh, lc[:, t], lh[:, t]
    if reverse:
        dU = dz[:, :T - 1].dot(h[:, 1:].T)
    else:
        dU = dz[:, 1:].dot(h[:, :T - 1].T)
    return dz, dU, dP


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
                 subsample=1, subsampleLayer=1, dropout=0.0, dropoutSeed=33, peephole=False, zoneoutCell=0.0,
                 zoneoutHidden=0.0, interLayer=0, interWeight=0.0, selfCondition=False, dtype=np.float64,
                 round_f32=True):
        hi = numLayers + 1 if allowTopTemporal else numLayers
        if numTemporal < 0:
            raise ValueError("numTemporal=%d must be >= 0" % numTemporal)
        if numTemporal > 1 and (temporalLayer <= 0 or temporalLayer + numTemporal - 1 >= hi):
            raise ValueError("numTemporal=%d from temporalLayer=%d does not fit" % (numTemporal, temporalLayer))
        if cell not in ("relu", "lstm"):
            raise ValueError("cell=%r" % (cell,))
        if not 0.0 <= dropout < 1.0:
            raise ValueError("dropout=%r must be in [0, 1)" % (dropout,))
        if peephole and cell != "lstm":
            raise ValueError("peephole=True needs cell='lstm'; cell is %r" % (cell,))
        for name, z in (("zoneoutCell", zoneoutCell), ("zoneoutHidden", zoneoutHidden)):
            if not 0.0 <= z < 1.0:
                raise ValueError("%s=%r must be in [0, 1)" % (name, z))
        if (zoneoutCell > 0.0 or zoneoutHidden > 0.0) and cell != "lstm":
            raise ValueError("zoneout needs cell='lstm'; cell is %r" % (cell,))
        self.inputDim, self.outputDim, self.layerSize, self.numLayers = inputDim, outputDim, layerSize, numLayers
        self.maxBatch, self.reg, self.dtype, self.round_f32 = maxBatch, reg, dtype, round_f32
        self.temporalLayer = temporalLayer if 0 < temporalLayer < hi else -1
        self.numTemporal = max(1, numTemporal) if self.temporalLayer > 0 else 0
        self.unidirectional, self.cell, self.layerNorm = bool(unidirectional), cell, bool(layerNorm)
        self.nrec = 1 if self.unidirectional else 2
        self.k, self.L = (int(subsample), int(subsampleLayer)) if subsample > 1 else (1, 0)
        self.dropout, self.dropoutSeed = float(dropout), int(dropoutSeed)
        self.dropoutStep, self.utt = 0, 0       # the masks' step and the minibatch index of the utterance computed
        self.peephole = bool(peephole)
        self.zoneoutCell, self.zoneoutHidden = float(zoneoutCell), float(zoneoutHidden)
        self.expectation = False                # zoneout's expectation (forward-only calls) in place of its masks
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
        self.selfCondition = bool(selfCondition)
        if self.selfCondition and not self.interLayer:
            raise ValueError("selfCondition=True needs interLayer >= 1")
        self.interCost, self.interSkip = 0.0, False
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

    def entries(self):
        """Number of [P, dummy] pairs: one per direction of every LSTM layer with peepholes."""
        return self.numTemporal * self.nrec if self.peephole else 0

    def peep_index(self, j, d):
        """Stack index of P of direction d of temporal layer j: behind the [gamma, beta] pairs."""
        return self.numLayers + 1 + self.numTemporal * self.nrec + len(self.normedLayers()) + j * self.nrec + d

    def weight_indices(self):
        """Stack indices of the matrices L2 regularises: the maps and the recurrent matrices."""
        return range(self.numLayers + 1 + self.numTemporal * self.nrec)

    def stacked(self, i):
        return self.k > 1 and i == self.L

    def lam(self):
        return float(np.float32(self.interWeight))

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
        out += [(H, 1), (H, 1)] * len(self.normedLayers())
        out += [(3, H), (1, 1)] * self.entries()
        return out + ([(H, self.outputDim), (H, 1)] if self.selfCondition else [])

    def initParams(self):
        """NNet.initParams's draws, rounded to float32: every matrix uniform in +-sqrt(6)/sqrt(rows+cols), biases 0,
        gamma 1 and beta 0, P, W_c and b_c 0, the last four without a draw."""
        shapes = self.shapes()
        nw = len(self.weight_indices())
        nln = nw + len(self.normedLayers())
        stack = []
        for t, ((m, n), bshape) in enumerate(zip(shapes[0::2], shapes[1::2])):
            if t <= self.numLayers:
                s = np.sqrt(6) / np.sqrt(n + m)
                stack.append([np.random.rand(m, n) * 2 * s - s, np.zeros(bshape)])
            elif t < nw:
                scale = np.sqrt(6) / np.sqrt(m + n)
                stack.append([2 * scale * np.random.rand(m, n) - scale, np.zeros(bshape)])
            else:
                stack.append([np.ones((m, n)) if t < nln else np.zeros((m, n)), np.zeros(bshape)])
        self.stack = [[w.astype(np.float32).astype(self.dtype), b.astype(self.dtype)] for w, b in stack]
        self.grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]

    def _keys(self, top):
        """Semantic key of every stack index, the output map counting as map `top`."""
        keys = [("map", i if i <= self.numLayers else top) for i in range(1, self.numLayers + 2)]
        keys += [("rec", j, d) for j in range(self.numTemporal) for d in range(self.nrec)]
        keys += [("ln", i) for i in self.normedLayers()]
        keys += [("peep", j, d) for j in range(self.numTemporal) for d in range(self.nrec)] if self.peephole else []
        return keys + ([("cond",)] if self.selfCondition else [])

    def head(self):
        """The head net of the intermediate loss over the same arrays: hidden layers 1..m (their temporal layers,
        normalisation, dropout and zoneout masks, and subsampling when it starts at or below m) and the output map; and
        the index of each of its stack entries in this net's stack."""
        m, tl = self.interLayer, self.temporalLayer
        nt = min(self.numTemporal, m - tl + 1) if self.numTemporal and tl <= m else 0
        sub = 0 < self.L <= m
        net = Net(self.inputDim, self.outputDim, self.layerSize, m, self.maxBatch, temporalLayer=tl if nt else -1,
                  unidirectional=self.unidirectional, numTemporal=nt, allowTopTemporal=True, cell=self.cell,
                  layerNorm=self.layerNorm, subsample=self.k if sub else 1, subsampleLayer=self.L if sub else 1,
                  dropout=self.dropout, dropoutSeed=self.dropoutSeed, peephole=self.peephole,
                  zoneoutCell=self.zoneoutCell, zoneoutHidden=self.zoneoutHidden, dtype=self.dtype,
                  round_f32=self.round_f32)
        full = {k: t for t, k in enumerate(self._keys(self.numLayers + 1))}
        index = [full[k] for k in net._keys(self.numLayers + 1)]
        net.stack = [self.stack[t] for t in index]
        net.dropoutStep, net.utt, net.expectation = self.dropoutStep, self.utt, self.expectation
        return net, index

    # ------------------------------------------------------------------ forward
    def drop(self, h, layer):
        """An (H, T) activation of hidden layer `layer` times mask * s, in h's dtype (s is the float32 scale, widened
        exactly)."""
        keep = keep_mask(self.dropout, self.dropoutSeed, self.dropoutStep, layer, self.utt, h.shape[1], h.shape[0]).T
        return np.where(keep, h * h.dtype.type(threshold_scale(self.dropout)[1]), h.dtype.type(0))

    def cell_args(self, j, d, T):
        """(P, lc, lh) of direction d of temporal layer j over T frames of the current utterance: its peephole weights
        and its zoneout lambdas (the drawn masks, or the expectation), zeros where the net has none."""
        H, dt = self.layerSize, self.dtype
        P = self.stack[self.peep_index(j, d)][0] if self.peephole else np.zeros((3, H), dtype=dt)
        if self.expectation:
            return (P, np.full((H, T), float(np.float32(self.zoneoutCell)), dtype=dt),
                    np.full((H, T), float(np.float32(self.zoneoutHidden)), dtype=dt))
        if self.zoneoutCell > 0.0 or self.zoneoutHidden > 0.0:
            lc, lh = zoneout_masks(self.zoneoutCell, self.zoneoutHidden, self.dropoutSeed, self.dropoutStep,
                                   self.temporalLayer + j, d, self.utt, T, H)
            return P, lc.T.astype(dt), lh.T.astype(dt)
        return P, np.zeros((H, T), dtype=dt), np.zeros((H, T), dtype=dt)

    def conditioned(self, hActs):
        """(X'_m, P) of the activations hActs: P = softmax(W_{N+1} X_m + b_{N+1}), X'_m = X_m + W_c P + b_c."""
        m, N = self.interLayer, self.numLayers
        P = self._softmax(self.stack[N][0].dot(hActs[m]) + self.stack[N][1]).astype(self.dtype)
        Wc, bc = self.stack[-1]
        return hActs[m] + Wc.dot(P) + bc, P

    def map_input(self, hActs, i, cond=None):
        """What affine map i reads: X_{i-1} (X'_m at map m + 1 of a self-conditioned net, cond[0] when given), or S
        stacked from it at map L."""
        x = hActs[i - 1]
        if self.selfCondition and i == self.interLayer + 1:
            x = (self.conditioned(hActs) if cond is None else cond)[0]
        return stack_frames(x, self.k) if self.stacked(i) else x

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
                j = i - self.temporalLayer
                idx = self.rec(j)
                if self.cell == "lstm":
                    gs, cs, hs = [], [], []
                    for d in range(self.nrec):
                        g, c, h = lstm_direction(z[d * 4 * H:(d + 1) * 4 * H], self.stack[idx[d]][0], d == 1,
                                                 *self.cell_args(j, d, T))
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
    def costAndGradGiven(self, data, labels, hActs, temporal, cond=None):
        """Back-propagation through GIVEN activations (X_1 .. X_{N+1} and each temporal layer's own, as `forward`
        returns them, and cond = (X'_m, P) of a self-conditioned net; e.g. the GPU's): the ReLU, clip and dropout masks
        are the given arrays' (X_i > 0), and each normalised layer's xh and rstd are recomputed in float64 from the
        given input of its map.  Without cond, X'_m and P are recomputed from the given X_m."""
        dt = self.dtype
        hActs = [np.asarray(data, dtype=dt)] + [np.asarray(x, dtype=dt) for x in hActs]
        cvt = lambda x: None if x is None else (np.asarray(x, dtype=dt) if not isinstance(x, list)  # noqa: E731
                                                 else [np.asarray(y, dtype=dt) for y in x])
        temporal = [tuple(cvt(x) for x in t) for t in temporal]
        cond = None if cond is None else tuple(np.asarray(x, dtype=dt) for x in cond)
        return self.costAndGrad(data, labels, _given=(hActs, temporal, self._softmax(hActs[-1])), _cond=cond)

    def costAndGrad(self, data, labels, _given=None, _cond=None):
        """(main cost, gradient of the objective, main skip) of one utterance; the intermediate nll and skip are left
        in interCost / interSkip."""
        hActs, temporal, probs = self.forward(data) if _given is None else _given
        cost, deltas, skip = brnn_oracle._ctc_loss(np.asfortranarray(probs.astype(np.float64)),
                                                   np.asarray(labels, dtype=np.int32))
        grad = [[np.zeros_like(w), np.zeros_like(b)] for w, b in self.stack]
        if self.reg > 0:
            self.regcost = sum((self.reg / 2.0) * float(np.sum(self.stack[k][0].astype(np.float64) ** 2))
                               for k in self.weight_indices())
            cost = cost + self.regcost
        if not skip:
            cond = _cond if _cond is not None or not self.selfCondition else self.conditioned(hActs)
            self._backprop(deltas, hActs, temporal, cond, grad)
            if self.reg > 0:
                for k in self.weight_indices():
                    grad[k][0] += self.reg * self.stack[k][0]
        if self.interLayer:
            self._add_head_gradient(data, labels, hActs, temporal, grad)
        self.grad = grad
        return cost, grad, skip

    def _backprop(self, deltas, hActs, temporal, cond, grad):
        """The main CTC's deltas back through every layer into grad."""
        H, dt, N = self.layerSize, self.dtype, self.numLayers
        deltasIn = (deltas.astype(np.float32) if self.round_f32 else deltas).astype(dt)
        for i in range(N, -1, -1):
            w = self.stack[i][0]
            grad[i][0] = deltasIn.dot(self.map_input(hActs, i + 1, cond).T)
            grad[i][1] = deltasIn.sum(axis=1)[:, None]
            if i == 0:
                break
            deltasOut = w.T.dot(deltasIn)
            if self.stacked(i + 1):
                deltasOut = unstack_frames(deltasOut, self.k, hActs[i].shape[1])
            if self.selfCondition and i == self.interLayer:     # D'_m through X'_m = X_m + W_c P + b_c
                P = cond[1]
                dP = self.stack[-1][0].T.dot(deltasOut)
                dA = P * (dP - (P * dP).sum(axis=0)[None, :])
                grad[-1][0] = deltasOut.dot(P.T)
                grad[-1][1] = deltasOut.sum(axis=1)[:, None]
                grad[N][0] = grad[N][0] + dA.dot(hActs[i].T)
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
                        dz, grad[idx[d]][0], dP = lstm_direction_bptt(deltasOut, gates[d * 4 * H:(d + 1) * 4 * H],
                                                                      cs[d], hs[d], self.stack[idx[d]][0], d == 1,
                                                                      *self.cell_args(j, d, T))
                        if self.peephole:
                            grad[self.peep_index(j, d)][0] = dP
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
                    xh, rstd = layer_norm(w_in.dot(self.map_input(hActs, i, cond)) + b_in)
                    g, grad[k][0], grad[k][1] = layer_norm_backward(g, self.stack[k][0], xh, rstd)
                deltasOut = g
            deltasIn = deltasOut

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

    def _add_head_gradient(self, data, labels, hActs, temporal, grad):
        """The intermediate term: lambda times the head net's gradient through the same X_1 .. X_m, added tensor by
        tensor unless the intermediate CTC skips."""
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

    def objective(self, data, labels):
        """nll_main (+ the L2 cost) + lambda nll_aux, the intermediate term left out where its CTC skips."""
        cost, _, _ = self.costAndGrad(data, labels)
        return cost + (0.0 if not self.interLayer or self.interSkip else self.lam() * self.interCost)

    def costAndGradBatch(self, datas, labelss, utts=None):
        """Per-utterance gradients summed, the L2 term added once to the weight matrices; utterance u draws the dropout
        and zoneout masks of minibatch index utts[u] (default u).  Each CTC skips on its own: an utterance the main
        CTC skips adds its intermediate gradient alone.  With the intermediate loss on, leaves the per-utterance
        intermediate nll and skips in interCosts / interSkips."""
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
        if self.interLayer:
            self.interCosts, self.interSkips = np.array(icosts), np.array(iskips)
        return np.array(costs), self.grad, np.array(skips)
