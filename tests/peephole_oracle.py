"""peephole_oracle.py -- TEST INFRASTRUCTURE ONLY: the float64 restatement of a net whose LSTM layers have peephole
connections (include/ctcb200.h: peephole = 1), built on tests/net_oracle.Net.

Per direction P = [p_i; p_f; p_o] (3 x H): i = sigmoid(z_i + p_i c_prev), f = sigmoid(z_f + p_f c_prev),
o = sigmoid(z_o + p_o c_t), with c_prev = c_{t-1} (c_{t+1} backward in time) and 0 before the first frame.  BPTT:
dz_o = dh tanh(c) o(1-o); dc = dh o (1 - tanh^2 c) + p_o dz_o + f_next dc_next + p_i dz_i,next + p_f dz_f,next;
dz_i, dz_f, dz_g from dc as without peepholes; dp_i = sum dz_i c_prev, dp_f = sum dz_f c_prev, dp_o = sum dz_o c.

PeepholeNet takes Net's keyword arguments plus peephole (default True; it needs cell='lstm').  Its stack is Net's
followed by [P, dummy] of every direction of every LSTM layer in the recurrent entries' order, P = 0 without a draw, so
initParams draws Net's numbers; P is not L2-regularised.  Its passes are Net's own, with the LSTM cell of each
direction replaced by the peephole cell of that direction's P: Net calls the cell functions of its module with the
direction's recurrent matrix U, and PeepholeNet routes each call, by U, to the P that belongs with it."""
import contextlib

import numpy as np

import net_oracle
from net_oracle import Net, _sig


def lstm_direction(P, U, reverse, peephole):
    """One direction over one utterance: P = [4H][T] pre-activations, U = 4H x H, peephole its 3 x H [p_i; p_f; p_o].
    Returns the activated gates [4H][T] (o after its peephole), c [H][T], h [H][T]."""
    H = U.shape[1]
    T = P.shape[1]
    gates = np.zeros_like(P)
    c = np.zeros((H, T), dtype=P.dtype)
    h = np.zeros((H, T), dtype=P.dtype)
    hp = np.zeros(H, dtype=P.dtype)
    cp = np.zeros(H, dtype=P.dtype)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        z = P[:, t] + U.dot(hp)
        i, f, g = _sig(z[:H] + peephole[0] * cp), _sig(z[H:2 * H] + peephole[1] * cp), np.tanh(z[2 * H:3 * H])
        cp = f * cp + i * g
        o = _sig(z[3 * H:] + peephole[2] * cp)
        hp = o * np.tanh(cp)
        gates[:, t] = np.concatenate([i, f, g, o])
        c[:, t], h[:, t] = cp, hp
    return gates, c, h


def lstm_direction_bptt(dh_in, gates, c, h, U, reverse, peephole):
    """BPTT of one direction given its activations: dh_in = [H][T] gradient w.r.t. the layer's output.  Returns dz
    [4H][T], dU and dP (3 x H)."""
    H = U.shape[1]
    T = dh_in.shape[1]
    dz = np.zeros_like(gates)
    dzn = np.zeros(4 * H, dtype=dh_in.dtype)
    dcn = np.zeros(H, dtype=dh_in.dtype)
    fn = np.zeros(H, dtype=dh_in.dtype)
    dP = np.zeros((3, H), dtype=dh_in.dtype)
    for t in (range(T) if reverse else range(T - 1, -1, -1)):
        i, f, g, o = gates[:H, t], gates[H:2 * H, t], gates[2 * H:3 * H, t], gates[3 * H:, t]
        dh = dh_in[:, t] + U.T.dot(dzn)
        tc = np.tanh(c[:, t])
        tp = t + 1 if reverse else t - 1
        cprev = c[:, tp] if 0 <= tp < T else np.zeros(H, dtype=dh_in.dtype)
        dzo = dh * tc * o * (1 - o)
        dc = dh * o * (1 - tc * tc) + peephole[2] * dzo + dcn * fn + peephole[0] * dzn[:H] + peephole[1] * dzn[H:2 * H]
        dz[:, t] = np.concatenate([dc * g * i * (1 - i), dc * cprev * f * (1 - f), dc * i * (1 - g * g), dzo])
        dP[0] += dz[:H, t] * cprev
        dP[1] += dz[H:2 * H, t] * cprev
        dP[2] += dzo * c[:, t]
        dzn, dcn, fn = dz[:, t], dc, f
    if reverse:
        dU = dz[:, :T - 1].dot(h[:, 1:].T)
    else:
        dU = dz[:, 1:].dot(h[:, :T - 1].T)
    return dz, dU, dP


class PeepholeNet(Net):
    def __init__(self, *args, peephole=True, **kw):
        Net.__init__(self, *args, **kw)
        if peephole and self.cell != "lstm":
            raise ValueError("peephole=True needs cell='lstm'; cell is %r" % (self.cell,))
        self.peephole = bool(peephole)

    def entries(self):
        """Number of [P, dummy] pairs behind Net's stack."""
        return self.numTemporal * self.nrec if self.peephole else 0

    def peep_index(self, j, d):
        """Stack index of P of direction d of temporal layer j: behind every tensor of Net's stack."""
        return len(Net.shapes(self)) // 2 + j * self.nrec + d

    def shapes(self):
        return Net.shapes(self) + [(3, self.layerSize), (1, 1)] * self.entries()

    def initParams(self):
        """Net's draws (the [P, dummy] pairs lie behind every drawn tensor), P = 0."""
        Net.initParams(self)
        for k in range(len(self.stack) - self.entries(), len(self.stack)):
            self.stack[k][0][...] = 0.0

    @contextlib.contextmanager
    def _cell(self):
        """Within it, net_oracle's LSTM cell functions are the peephole cell of the direction whose U they are given;
        the BPTT leaves dP of each direction in self._dP, by stack index."""
        if not self.peephole:
            yield
            return
        which = {}
        for j in range(self.numTemporal):
            for d, r in enumerate(self.rec(j)[:self.nrec]):
                which[id(self.stack[r][0])] = self.peep_index(j, d)
        saved = net_oracle.lstm_direction, net_oracle.lstm_direction_bptt

        def fwd(P, U, reverse):
            return lstm_direction(P, U, reverse, self.stack[which[id(U)]][0])

        def bwd(dh_in, gates, c, h, U, reverse):
            k = which[id(U)]
            dz, dU, self._dP[k] = lstm_direction_bptt(dh_in, gates, c, h, U, reverse, self.stack[k][0])
            return dz, dU

        net_oracle.lstm_direction, net_oracle.lstm_direction_bptt = fwd, bwd
        try:
            yield
        finally:
            net_oracle.lstm_direction, net_oracle.lstm_direction_bptt = saved

    def forward(self, data):
        with self._cell():
            return Net.forward(self, data)

    def costAndGrad(self, data, labels, _given=None):
        self._dP = {}
        with self._cell():
            cost, grad, skip = Net.costAndGrad(self, data, labels, _given)
        for k, dP in self._dP.items():
            grad[k][0] = dP
        return cost, grad, skip
