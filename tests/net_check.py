"""net_check.py -- TEST INFRASTRUCTURE ONLY: a device net's last training call against tests/net_oracle.Net.

compare() reads what the device left behind -- per-utterance costs and skips, the gradient, and every activation
array ctcb_brnn_activation_offset exposes -- and runs one loop over the utterances: the oracle's own forward and
back-propagation (its own float64 masks), and its back-propagation through the device's own activations (the device's
masks, and X'_m and P of a self-conditioned net), each summed over the utterances under Net.costAndGradBatch's rule
with reg * W added once.  It returns plain numbers; the tests decide which bounds apply."""
import ctypes

import numpy as np

from net_oracle import frames, stack_frames


def rel(a, b):
    """Relative Frobenius error of a against b (0 if both are 0, inf if only b is)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nb = np.linalg.norm(b)
    if nb == 0.0:
        return 0.0 if np.linalg.norm(a) == 0.0 else float("inf")
    return float(np.linalg.norm(a - b) / nb)


def relmax(a, b):
    """Largest element-wise error of a against b relative to b's largest magnitude."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


def workspace_activations(nn, B, Tmax):
    """{(what, layer): float32 [T][B][width]} of every array the activation hook exposes for nn's last call of B
    utterances of at most Tmax frames (what 0 X, 1 For / h_f, 2 Back / h_b, 3 gates, 4 c_f, 5 c_b, 6 S, and with
    selfCondition 12 X'_m and 13 P), each at its map's own frame count: ceil(Tmax / k) from map L = subsampleLayer up
    (X'_m and P at layer m's)."""
    from _ctcb import lib
    off, width = ctypes.c_size_t(), ctypes.c_int32()
    out = {}
    for what in list(range(7)) + ([12, 13] if nn.selfCondition else []):
        for layer in range(nn.numLayers + 2):
            if lib.ctcb_brnn_activation_offset(ctypes.byref(nn._cfg), what, layer, ctypes.byref(off),
                                               ctypes.byref(width)) != 0:
                continue
            rate = nn.interLayer if what >= 12 else layer
            T = nn.frames(Tmax) if what == 6 or (nn.subsample > 1 and rate >= nn.subsampleLayer) else Tmax
            n = T * B * width.value
            out[what, layer] = nn._ws[off.value:off.value + 4 * n].view(nn._torch.float32).cpu().numpy() \
                .reshape(T, B, width.value)
    return out


def compare(nn, oracle, datas, labelss, lens, utts=None):
    """The device net nn, after a training call on (datas, labelss) of lengths lens in one micro-batch, against
    oracle (the same parameters, the same dropout step; its reg is the device's).  Utterance u draws the dropout mask
    of minibatch index utts[u] (default u).  Returns a dict:
      acts         workspace_activations of the call
      skips        the device's skips; skips_own / skips_given the oracle's on its own and on the device's activations
      cost_own     largest relative error of the device's costs against the oracle's own (non-skipped utterances)
      cost_given   the same against the oracle's costs on the device's activations
      inter_cost, inter_skips, inter_skips_own (interLayer only)
                   largest relative error of the device's intermediate nll against the oracle's own (utterances the
                   device's intermediate CTC keeps), the device's intermediate skips and the oracle's own
      fwd          {kind: largest relmax over the utterances}: X (list, layers 1..N+1, each layer's output: For of a
                   uni-directional clipped-ReLU layer, h_f + h_b of an LSTM layer), For and Back (clipped-ReLU), gates,
                   h and c (LSTM), S (subsampling)
      grad_given, grad_given_elem, grad_plain
                   per tensor of the flat order (w_0, b_0, w_1, ...): rel and relmax of the device's gradient against
                   the back-propagation through its activations, and rel against the oracle's own gradient; 0 where
                   the oracle's given gradient is exactly 0, which the device's must then be too."""
    B = len(datas)
    Tmax = max(lens)
    acts = workspace_activations(nn, B, Tmax)
    costs = nn._cost[:B].cpu().numpy().astype(np.float64)
    skips = nn._skip[:B].cpu().numpy() != 0
    grad = [x.cpu().numpy().astype(np.float64) for g in nn.grad for x in g]
    N, k, L = oracle.numLayers, oracle.k, oracle.L
    lstm = oracle.cell == "lstm"
    temporal = [i for i in range(1, N + 2) if oracle.temporal(i)]
    reg, oracle.reg = oracle.reg, 0.0
    own = [[np.zeros_like(w), np.zeros_like(b)] for w, b in oracle.stack]
    given = [[np.zeros_like(w), np.zeros_like(b)] for w, b in oracle.stack]
    c_own, c_given, s_own, s_given, i_own, i_skip = [], [], [], [], [], []
    fwd = dict(X=[0.0] * (N + 1))
    kinds = (["h", "c", "gates"] if lstm else ["For"] + ([] if oracle.unidirectional else ["Back"])) if temporal else []
    fwd.update((kind, 0.0) for kind in kinds + (["S"] if k > 1 else []))
    try:
        for u, (d, l) in enumerate(zip(datas, labelss)):
            oracle.utt = u if utts is None else utts[u]
            hActs, o_temp, probs = oracle.forward(d)
            g_acts, g_temp = [], []
            for i in range(1, N + 2):
                Tu = frames(lens[u], k) if i >= L > 0 else lens[u]
                a = lambda what, layer=i: acts[what, layer][:Tu, u].T      # noqa: E731
                act = a(0)
                if i in temporal:
                    ot = o_temp[i - temporal[0]]
                    dirs = [1] + ([] if oracle.unidirectional else [2])
                    if lstm:
                        gh, gc = [a(w) for w in dirs], [a(w + 3) for w in dirs]
                        g_temp.append((act, gc, gh))
                        fwd["gates"] = max(fwd["gates"], relmax(act, ot[0]))
                        fwd["c"] = max([fwd["c"]] + [relmax(x, y) for x, y in zip(gc, ot[1])])
                        fwd["h"] = max([fwd["h"]] + [relmax(x, y) for x, y in zip(gh, ot[2])])
                        act = sum(x.astype(np.float64) for x in gh)
                    else:
                        sweeps = [a(w) for w in dirs]
                        for kind, x, y in zip(("For", "Back"), sweeps, ot):
                            fwd[kind] = max(fwd[kind], relmax(x, y))
                        g_temp.append((sweeps[0], sweeps[1] if len(sweeps) > 1 else None))
                        if oracle.unidirectional:
                            act = sweeps[0]
                g_acts.append(act)
                fwd["X"][i - 1] = max(fwd["X"][i - 1], relmax(act, hActs[i]))
            if k > 1:
                fwd["S"] = max(fwd["S"], relmax(acts[6, 0][:frames(lens[u], k), u].T, stack_frames(hActs[L - 1], k)))
            cond = None
            if oracle.selfCondition:
                Tm = frames(lens[u], k) if oracle.interLayer >= L > 0 else lens[u]
                cond = (acts[12, 0][:Tm, u].T, acts[13, 0][:Tm, u].T)
            for path, tot, c_, s_ in (((hActs, o_temp, probs), own, c_own, s_own), (None, given, c_given, s_given)):
                if path is None:
                    c, g, s = oracle.costAndGradGiven(d, l, g_acts, g_temp, cond=cond)
                else:
                    c, g, s = oracle.costAndGrad(d, l, _given=path)
                    i_own.append(oracle.interCost)
                    i_skip.append(oracle.interSkip)
                c_.append(c)
                s_.append(bool(s))
                for (tw, tb), (gw, gb) in zip(tot, g):     # a main skip adds the intermediate gradient alone
                    tw += gw
                    tb += gb
    finally:
        oracle.reg = reg
    for tot in (own, given):
        for t in oracle.weight_indices():
            tot[t][0] += reg * oracle.stack[t][0]
    own, given = [x for g in own for x in g], [x for g in given for x in g]
    grad_given, grad_elem, grad_plain = [], [], []
    for x, y, z in zip(grad, given, own):
        x = x.reshape(y.shape)
        if not np.any(y):
            assert not np.any(x), "the oracle's gradient is exactly 0 where the device's is not"
            grad_given.append(0.0)
            grad_elem.append(0.0)
            grad_plain.append(0.0)
            continue
        grad_given.append(rel(x, y))
        grad_elem.append(relmax(x, y))
        grad_plain.append(rel(x, z))
    cost_err = lambda got, ref, ok: float(np.max(np.abs(got[ok] - np.array(ref)[ok]) / np.abs(np.array(ref)[ok]))) \
        if ok.any() else 0.0     # noqa: E731
    out = dict(acts=acts, skips=skips, skips_own=np.array(s_own), skips_given=np.array(s_given),
               cost_own=cost_err(costs, c_own, ~skips), cost_given=cost_err(costs, c_given, ~skips), fwd=fwd,
               grad_given=grad_given, grad_given_elem=grad_elem, grad_plain=grad_plain)
    if oracle.interLayer:
        iskips = np.asarray(nn.interSkips[:B], dtype=bool)
        out.update(inter_cost=cost_err(np.asarray(nn.interCosts[:B], np.float64), i_own, ~iskips), inter_skips=iskips,
                   inter_skips_own=np.array(i_skip))
    return out
