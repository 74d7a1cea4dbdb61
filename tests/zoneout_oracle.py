"""zoneout_oracle.py -- TEST INFRASTRUCTURE ONLY: the float64 restatement of a net whose LSTM layers have zoneout
(include/ctcb200.h: zoneout = 1), built on tests/peephole_oracle.PeepholeNet, so zoneout composes with peepholes.

The masks: unit j of frame t (0..T-1, at the layer's rate) of minibatch utterance g in direction d of temporal layer i
(its hidden-layer index) at step s draws
    (r0, r1, r2, r3) = Philox4x32-10(counter = (s mod 2^32, g mod 2^32, t, (i << 24) | (d << 23) | j),
                                     key = (seed mod 2^32, seed >> 32))
and lambda_c = 1 iff r0 < floor(z_c 2^32), lambda_h = 1 iff r1 < floor(z_h 2^32) (float64 products, z the float32 the
library is given).  The expectation (forward-only calls) is lambda_c = float32(z_c), lambda_h = float32(z_h).
Forward, per direction:  c~ = f c_prev + i g;  c = lc c_prev + (1 - lc) c~;  h~ = o tanh(c);  h = lh h_prev + (1 - lh) h~
(peepholes: i, f see the zoned c_prev, o the zoned c).  BPTT ("next" = the step after t in the direction's order):
    dh = delta + U^T dz_next + lh_next dh_next;  dh~ = (1 - lh) dh;  dz_o = dh~ tanh(c) o(1-o)
    dc = dh~ o (1 - tanh^2 c) [+ p_o dz_o] + (lc_next + (1 - lc_next) f_next) dc_next [+ p_i dz_i,next + p_f dz_f,next]
    dc~ = (1 - lc) dc;  dz_i = dc~ g i(1-i);  dz_f = dc~ c_prev f(1-f);  dz_g = dc~ i(1-g^2)
With lambda = 0 every formula reduces, operation for operation, to net_oracle's (peephole=False) or peephole_oracle's
cell, so at z = 0 ZoneoutNet equals Net / PeepholeNet bit for bit.

ZoneoutNet takes PeepholeNet's keyword arguments (peephole defaults to False here) plus zoneoutCell and zoneoutHidden;
its attribute `expectation` (default False) switches its passes to the expectation cell.  The masks follow
dropoutSeed, dropoutStep and utt, as dropout's do.  Net and PeepholeNet are unchanged."""
import contextlib

import numpy as np

import net_oracle
from net_oracle import _sig, philox4x32_10
from peephole_oracle import PeepholeNet


def threshold(z):
    """floor(z 2^32) of the float32 z the library is given, in float64."""
    return int(np.floor(float(np.float32(z)) * 4294967296.0))


def draws(seed, step, layer, d, g, T, H):
    """Philox outputs (T, H, 4) uint32 of units 0..H-1 of frames 0..T-1 of minibatch utterance g, direction d of
    temporal layer `layer`, at `step`."""
    t, j = np.meshgrid(np.arange(T, dtype=np.uint64), np.arange(H, dtype=np.uint64), indexing="ij")
    ctr = np.stack([np.full_like(t, int(step) & 0xFFFFFFFF), np.full_like(t, int(g) & 0xFFFFFFFF), t,
                    np.uint64((int(layer) << 24) | (int(d) << 23)) | j], axis=-1)
    return philox4x32_10(ctr, (int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF))


def masks(zc, zh, seed, step, layer, d, g, T, H):
    """Boolean (T, H) lambda_c and lambda_h of one direction of one utterance (True: keep the previous value)."""
    r = draws(seed, step, layer, d, g, T, H)
    return r[..., 0] < np.uint32(threshold(zc)), r[..., 1] < np.uint32(threshold(zh))


def lstm_direction(P, U, reverse, peephole, lc, lh):
    """One direction over one utterance with zoneout: P = [4H][T] pre-activations, U = 4H x H, peephole its
    [p_i; p_f; p_o] or None, lc / lh [H][T] the lambdas.  Returns the activated gates [4H][T], c [H][T], h [H][T]
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
        if peephole is None:
            i, f, g = _sig(z[:H]), _sig(z[H:2 * H]), np.tanh(z[2 * H:3 * H])
        else:
            i, f, g = _sig(z[:H] + peephole[0] * cp), _sig(z[H:2 * H] + peephole[1] * cp), np.tanh(z[2 * H:3 * H])
        cp = lc[:, t] * cp + (1 - lc[:, t]) * (f * cp + i * g)
        o = _sig(z[3 * H:]) if peephole is None else _sig(z[3 * H:] + peephole[2] * cp)
        hp = lh[:, t] * hp + (1 - lh[:, t]) * (o * np.tanh(cp))
        gates[:, t] = np.concatenate([i, f, g, o])
        c[:, t], h[:, t] = cp, hp
    return gates, c, h


def lstm_direction_bptt(dh_in, gates, c, h, U, reverse, peephole, lc, lh):
    """BPTT of one direction with zoneout given its activations.  Returns dz [4H][T], dU and dP (3 x H; zeros
    without peepholes)."""
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
        if peephole is None:
            dc = dht * o * (1 - tc * tc) + carry
        else:
            dc = dht * o * (1 - tc * tc) + peephole[2] * dzo + carry + peephole[0] * dzn[:H] + peephole[1] * dzn[H:2 * H]
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


class ZoneoutNet(PeepholeNet):
    def __init__(self, *args, peephole=False, zoneoutCell=0.0, zoneoutHidden=0.0, **kw):
        PeepholeNet.__init__(self, *args, peephole=peephole, **kw)
        for name, z in (("zoneoutCell", zoneoutCell), ("zoneoutHidden", zoneoutHidden)):
            if not 0.0 <= z < 1.0:
                raise ValueError("%s=%r must be in [0, 1)" % (name, z))
        if (zoneoutCell > 0.0 or zoneoutHidden > 0.0) and self.cell != "lstm":
            raise ValueError("zoneout needs cell='lstm'; cell is %r" % (self.cell,))
        self.zoneoutCell, self.zoneoutHidden = float(zoneoutCell), float(zoneoutHidden)
        self.expectation = False

    def lambdas(self, layer, d, T):
        """(lc, lh), each [H][T] in the net's dtype, of direction d of temporal layer `layer` for the current
        utterance: the drawn masks, or the expectation."""
        H, dt = self.layerSize, self.dtype
        if self.expectation:
            return (np.full((H, T), float(np.float32(self.zoneoutCell)), dtype=dt),
                    np.full((H, T), float(np.float32(self.zoneoutHidden)), dtype=dt))
        lc, lh = masks(self.zoneoutCell, self.zoneoutHidden, self.dropoutSeed, self.dropoutStep, layer, d, self.utt,
                       T, H)
        return lc.T.astype(dt), lh.T.astype(dt)

    @contextlib.contextmanager
    def _cell(self):
        """Within it, net_oracle's LSTM cell functions are the zoneout cell (with the peephole cell's P when the net
        has peepholes) of the direction whose U they are given; the BPTT leaves dP in self._dP, by stack index."""
        which = {}
        for j in range(self.numTemporal):
            for d, r in enumerate(self.rec(j)[:self.nrec]):
                which[id(self.stack[r][0])] = (self.temporalLayer + j, d,
                                               self.peep_index(j, d) if self.peephole else None)
        saved = net_oracle.lstm_direction, net_oracle.lstm_direction_bptt

        def fwd(P, U, reverse):
            layer, d, k = which[id(U)]
            lc, lh = self.lambdas(layer, d, P.shape[1])
            return lstm_direction(P, U, reverse, None if k is None else self.stack[k][0], lc, lh)

        def bwd(dh_in, gates, c, h, U, reverse):
            layer, d, k = which[id(U)]
            lc, lh = self.lambdas(layer, d, dh_in.shape[1])
            dz, dU, dP = lstm_direction_bptt(dh_in, gates, c, h, U, reverse, None if k is None else self.stack[k][0],
                                             lc, lh)
            if k is not None:
                self._dP[k] = dP
            return dz, dU

        net_oracle.lstm_direction, net_oracle.lstm_direction_bptt = fwd, bwd
        try:
            yield
        finally:
            net_oracle.lstm_direction, net_oracle.lstm_direction_bptt = saved
