"""CPU tests of the float64 restatement of the net (tests/net_oracle.py): with every feature off it is the pinned oracle
(oracle/brnn_oracle.py), it draws the library's tensor table, its gradient is the central difference of its cost for
every feature (stacked, uni-directional, DNN, dropout, LSTM, layer norm, subsampling) and for nets that combine
peepholes, zoneout and the intermediate or self-conditioned CTC (each feature alone is in its own CPU file), and
back-propagation through
given activations is the same as through its own; its LSTM cell and normalisation are torch's and its subsampled
nets torch autograd's.  No compute call is made on a device here."""
import ctypes

import numpy as np
import pytest

import recipes
from net_oracle import (Net, frames, layer_norm, layer_norm_backward, lstm_direction, lstm_direction_bptt,
                        stack_frames, unstack_frames)
from oracle import brnn_oracle


# ------------------------------------------------------------------------------------------- the pinned oracle
@pytest.mark.parametrize("kind", ["bi", "uni", "dnn"])
def test_every_feature_off_is_the_pinned_oracle(kind):
    """The same draws bit for bit, costs and every gradient within 1e-12."""
    datas, labelss = recipes.synth_batch(13, 11, [20, 17, 9], [5, 4, 3], seed=1)
    kw = dict(temporalLayer=-1 if kind == "dnn" else 2, reg=1e-3 * (kind != "uni"), unidirectional=kind == "uni")
    outs = []
    for cls in (Net, brnn_oracle.NNet):
        np.random.seed(5)
        nn = cls(13, 11, 32, 3, 20, **kw)
        nn.initParams()
        costs, grad, skips = nn.costAndGradBatch(datas, labelss)
        outs.append((costs, [np.array(x) for g in grad for x in g], nn.stack))
    (c1, g1, s1), (c2, g2, s2) = outs
    assert len(s1) == len(s2) and all(np.array_equal(a[0], b[0]) for a, b in zip(s1, s2))
    assert np.allclose(c1, c2, rtol=1e-12, atol=0)
    for a, b in zip(g1, g2):
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max())


def test_stacked_restatement_draws_the_extra_matrices_after_todays():
    np.random.seed(33)
    one = Net(13, 11, 16, 4, 20, temporalLayer=1, numTemporal=1)
    one.initParams()
    np.random.seed(33)
    three = Net(13, 11, 16, 4, 20, temporalLayer=1, numTemporal=3)
    three.initParams()
    assert len(three.stack) == len(one.stack) + 4
    for (a, _), (b, _) in zip(one.stack, three.stack):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------- the tensor table
def _table(D, K, H, N, tl, T, B, L, uni=0, nt=1, cell=0, ln=0, k=1, sl=1):
    import _ctcb
    from _ctcb import lib
    cfg = _ctcb.BrnnConfig(D, K, H, N, tl, T, B, L, 0.0, 20.0, uni, nt, cell, ln, k, sl)
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for i in range(lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))):
        assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        out.append((r.value, c.value))
    return out


# (D, K, H, N, tl, T, B, L, uni, nt, cell, ln, k, sl): LSTM stacks, layer-normalised nets (C2, a stack, a DNN, an LSTM
# net, a uni-directional net with odd H), W_L of every width at every map
SHAPES = [(13, 11, 70, 4, 2, 60, 8, 20, uni, nt, 1, 0, 1, 1) for uni in (0, 1) for nt in (1, 2, 3)] + \
    [(41, 62, 512, 2, 1, 200, 32, 30, 0, 1, 0, 1, 1, 1), (13, 11, 70, 4, 2, 37, 5, 9, 0, 2, 0, 1, 1, 1),
     (13, 11, 64, 3, 0, 40, 4, 9, 0, 1, 0, 1, 1, 1), (13, 11, 64, 3, 2, 60, 8, 20, 1, 1, 1, 1, 1, 1),
     (41, 32, 1824, 5, 3, 50, 4, 20, 1, 1, 0, 1, 1, 1)] + \
    [(13, 11, 64, 3, 2, 60, 8, 9, 0, 1, 0, 0, k, sl) for k in (2, 3, 4) for sl in (1, 2, 3, 4)]


@pytest.mark.parametrize("net", SHAPES)
def test_shapes_are_the_library_table(net):
    """shapes() is the library's tensor table, and initParams draws those shapes."""
    D, K, H, N, tl, T, B, L, uni, nt, cell, ln, k, sl = net
    o = Net(D, K, H, N, T, temporalLayer=tl, numTemporal=nt, unidirectional=bool(uni), allowTopTemporal=True,
            cell=("lstm" if cell else "relu"), layerNorm=bool(ln), subsample=k, subsampleLayer=sl)
    assert o.shapes() == _table(*net)
    o.initParams()
    assert [s for w, b in o.stack for s in (w.shape, b.shape)] == o.shapes()


# ------------------------------------------------------------------------------------------- finite differences
def _probe(net, x, idx, cost):
    """Central difference of cost() in entry idx of x, with eps = 1e-6."""
    eps = 1e-6
    old = x[idx]
    x[idx] = old + eps
    cp = cost()
    x[idx] = old - eps
    cm = cost()
    x[idx] = old
    return (cp - cm) / (2 * eps)


def _gradcheck_one(net, seed, probes):
    """The recipe of rnnetcpu.py:181-190 / tests/test_oracle.py: one utterance, `probes` entries of every matrix and one
    of every map's bias, |analytic - numeric| < 1e-4."""
    rng = np.random.RandomState(seed)
    np.random.seed(seed)
    net.initParams()
    if net.dropout:
        net.dropoutStep, net.utt = 3, 2
    data = rng.randn(net.inputDim, net.maxBatch)
    labels = np.array([1, 2, 2, 4], dtype=np.int32)
    cost, grad, skip = net.costAndGrad(data, labels)
    assert not skip
    grad = [[dw.copy(), db.copy()] for dw, db in grad]
    assert len(net.stack) == net.numLayers + 1 + net.numTemporal * net.nrec
    if net.dropout:     # the mask drops units of every ReLU hidden layer and changes the cost
        hActs = net.forward(data)[0]
        dropped = [i for i in range(1, net.numLayers + 1) if net.dropped(i)]
        assert dropped and all((hActs[i] == 0).mean() > 0.3 for i in dropped)
        p, net.dropout = net.dropout, 0.0
        assert abs(net.costAndGrad(data, labels)[0] - cost) > 1e-3
        net.dropout = p
    f = lambda: net.costAndGrad(data, labels)[0]        # noqa: E731
    for pi, (w, b) in enumerate(net.stack):
        for _ in range(probes):
            i, j = rng.randint(w.shape[0]), rng.randint(w.shape[1])
            num = _probe(net, w, (i, j), f)
            assert abs(grad[pi][0][i, j] - num) < 1e-4, (pi, i, j)
        if pi <= net.numLayers:     # the biases of the affine maps as well
            i = rng.randint(b.shape[0])
            assert abs(grad[pi][1][i, 0] - _probe(net, b, (i, 0), f)) < 1e-4, (pi, i)
    if not net.dropout:     # the recurrent gradients are not trivially zero (the probes would then prove nothing)
        assert all(np.abs(grad[r][0]).max() > 1e-6 for r in range(net.numLayers + 1, len(net.stack)))


def _gradcheck_batch(net, lens, nlabs, rng_seed, scale=1.0, every_pair_entry=False):
    """A ragged batch, reg > 0, weights times `scale`, gamma, beta moved off 1, 0 and P, W_c, b_c off 0: 3 entries of
    every tensor (every entry of the tensors behind the recurrent ones with every_pair_entry, one more in each sub-frame
    block of W_L) against the central difference of the summed objective (main + lambda intermediate),
    |analytic - numeric| <= 1e-6 max(1, |numeric|)."""
    np.random.seed(11)
    net.initParams()
    for w, _ in net.stack:
        w *= scale
    rng = np.random.RandomState(rng_seed)
    for i in net.normedLayers():
        gamma, beta = net.stack[net.ln_index(i)]
        gamma += 0.3 * rng.randn(*gamma.shape)
        beta += 0.3 * rng.randn(*beta.shape)
    for w, b in net.stack[net.peep_index(0, 0):]:      # [P, dummy] and [W_c, b_c], behind the [gamma, beta] pairs
        w[...] = rng.uniform(-0.5, 0.5, w.shape)
        if b.shape != (1, 1):
            b[...] = rng.uniform(-0.1, 0.1, b.shape)
    datas, labels = recipes.synth_batch(net.inputDim, net.outputDim, lens, nlabs, seed=3)
    _, grad, skips = net.costAndGradBatch(datas, labels)
    assert not skips.any() and not (net.interLayer and net.interSkips.any())
    N = net.numLayers
    base = N + 1 + net.numTemporal * net.nrec
    if net.layerNorm:
        assert len(net.stack) - base == len(net.normedLayers()) + net.entries() + net.selfCondition
        assert len(net.normedLayers()) > 0

    def f():
        costs = net.costAndGradBatch(datas, labels)[0]
        inter = net.lam() * net.interCosts.sum() if net.interLayer else 0.0
        return costs.sum() + net.regcost + inter
    for ti, (w, b) in enumerate(net.stack):
        for x, gx in ((w, grad[ti][0]), (b, grad[ti][1])):
            if N < ti < base and x is b:        # the recurrent matrices' dummies take no part
                continue
            idxs = list(np.ndindex(x.shape)) if every_pair_entry and ti >= base else \
                [tuple(rng.randint(0, s) for s in x.shape) for _ in range(3)]
            if net.stacked(ti + 1) and x is w:  # one entry in every sub-frame block of W_L
                n = x.shape[1] // net.k
                idxs += [(rng.randint(0, x.shape[0]), m * n + rng.randint(0, n)) for m in range(net.k)]
            for idx in idxs:
                num = _probe(net, x, idx, f)
                assert abs(num - gx[idx]) <= 1e-6 * max(1.0, abs(num)), (ti, idx, num, gx[idx])


# name: (Net arguments, recipe); every net in float64 without float32 hand-offs, reg = 1e-3
FD = {}
for _k in (2, 3):
    for _uni in (False, True):
        FD["stack_k%d_%s" % (_k, "uni" if _uni else "bi")] = (
            dict(dims=(7, 5, 12, 4, 9), temporalLayer=1, numTemporal=_k, unidirectional=_uni),
            dict(recipe="one", seed=3 + _k, probes=6))
for _name, _kw in {"bi": dict(N=3, temporalLayer=2), "uni": dict(N=3, temporalLayer=2, unidirectional=True),
                   "dnn": dict(N=3, temporalLayer=0), "relu_around_one_temporal": dict(N=4, temporalLayer=2),
                   "relu_around_two_temporal": dict(N=5, temporalLayer=2, numTemporal=2)}.items():
    _N = _kw.pop("N")
    FD["dropout_" + _name] = (dict(dims=(7, 5, 12, _N, 9), dropout=0.3, dropoutSeed=5, **_kw),
                              dict(recipe="one", seed=11, probes=5))
for _k in (1, 2, 3):
    for _uni in (False, True):      # k stacked LSTM layers between ReLU layers, saturated somewhat by larger weights
        FD["lstm_k%d_%s" % (_k, "uni" if _uni else "bi")] = (
            dict(dims=(5, 6, 4, _k + 2, 7), temporalLayer=2, numTemporal=_k, unidirectional=_uni, cell="lstm"),
            dict(recipe="batch", lens=[7, 4], nlabs=[3, 2], rng_seed=0, scale=2.0))
for _name, _c in {"bi": dict(tl=2, k=1), "uni": dict(tl=2, k=1, uni=True), "dnn": dict(tl=0, k=0),
                  "stack2": dict(tl=2, k=2, N=4), "lstm": dict(tl=2, k=1, cell="lstm"),
                  "bi_dropout": dict(tl=2, k=1, p=0.3)}.items():
    FD["layernorm_" + _name] = (
        dict(dims=(5, 6, 6, _c.get("N", 3), 8), temporalLayer=_c["tl"], numTemporal=_c["k"], layerNorm=True,
             unidirectional=bool(_c.get("uni")), cell=_c.get("cell", "relu"), dropout=_c.get("p", 0.0), dropoutSeed=5),
        dict(recipe="batch", lens=[7, 4], nlabs=[3, 2], rng_seed=2, every_pair_entry=True))
# subsampling: N, tl, nt, k, L, extra
SUBSAMPLE = {
    "bi_L1_k2": (3, 2, 1, 2, 1, {}),
    "bi_Ltl_k3": (3, 2, 1, 3, 2, {}),
    "uni_stack_inside_k2": (4, 2, 2, 2, 3, dict(uni=True)),
    "bi_stack_inside_k3": (4, 2, 2, 3, 3, {}),
    "bi_above_k2_ln_drop": (3, 1, 1, 2, 3, dict(ln=True, p=0.3)),
    "bi_top_k3": (3, 2, 1, 3, 4, {}),
    "dnn_k2_ln": (2, 0, 0, 2, 2, dict(ln=True)),
    "dnn_L1_k3_drop": (2, 0, 0, 3, 1, dict(p=0.25)),
    "lstm_bi_Ltl_k2": (3, 2, 1, 2, 2, dict(cell="lstm")),
    "lstm_uni_above_k3": (3, 1, 1, 3, 2, dict(cell="lstm", uni=True, ln=True)),
}
# ragged lengths, none a multiple of 2 or 3 but one; every T mod k
LENS, NLABS = [13, 8, 11, 7], [3, 2, 2, 1]


def _subsampled(name, **kw):
    N, tl, nt, k, L, x = SUBSAMPLE[name]
    return dict(dims=(5, 6, 6, N, 40), temporalLayer=tl, numTemporal=nt, subsample=k, subsampleLayer=L,
                dropout=x.get("p", 0.0), dropoutSeed=5, cell=x.get("cell", "relu"), unidirectional=bool(x.get("uni")),
                layerNorm=bool(x.get("ln")), **kw)


for _name in SUBSAMPLE:
    FD["subsample_" + _name] = (_subsampled(_name), dict(recipe="batch", lens=LENS, nlabs=NLABS, rng_seed=2))
# feature combinations: every tensor, P, W_c and b_c in full
FD["combo_bi_lstm_peep_zoneout_selfcond_ln_drop"] = (
    dict(dims=(5, 6, 6, 3, 13), temporalLayer=2, cell="lstm", peephole=True, zoneoutCell=0.3, zoneoutHidden=0.2,
         interLayer=2, interWeight=0.7, selfCondition=True, layerNorm=True, dropout=0.3, dropoutSeed=5),
    dict(recipe="batch", lens=LENS, nlabs=NLABS, rng_seed=2, every_pair_entry=True))
FD["combo_uni_lstm_zoneout_inter_sub_below"] = (
    dict(dims=(5, 6, 6, 4, 13), temporalLayer=2, numTemporal=2, unidirectional=True, cell="lstm", zoneoutCell=0.3,
         zoneoutHidden=0.2, interLayer=2, interWeight=0.7, subsample=2, subsampleLayer=1, dropoutSeed=5),
    dict(recipe="batch", lens=LENS, nlabs=NLABS, rng_seed=2, every_pair_entry=True))
FD["combo_bi_lstm_peep_zoneout_k2_selfcond_top"] = (
    dict(dims=(5, 6, 6, 4, 13), temporalLayer=2, numTemporal=2, cell="lstm", peephole=True, zoneoutCell=0.2,
         zoneoutHidden=0.3, interLayer=3, interWeight=0.5, selfCondition=True, dropout=0.2, dropoutSeed=5),
    dict(recipe="batch", lens=LENS, nlabs=NLABS, rng_seed=2, every_pair_entry=True))


@pytest.mark.parametrize("name", list(FD))
def test_oracle_gradient_matches_central_differences(name):
    kw, recipe = dict(FD[name][0]), dict(FD[name][1])
    net = Net(*kw.pop("dims"), reg=1e-3, round_f32=False, **kw)
    if recipe.pop("recipe") == "one":
        _gradcheck_one(net, **recipe)
    else:
        _gradcheck_batch(net, **recipe)


# ------------------------------------------------------------------------------------------- given activations
# every feature but dropout alone, which tests/test_dropout_cpu.py checks the same way
GIVEN = {
    "stack_uni": dict(N=5, temporalLayer=2, numTemporal=2, unidirectional=True),
    "dnn": dict(temporalLayer=-1),
    "lstm": dict(temporalLayer=2, numTemporal=2, cell="lstm"),
    "layernorm_dropout": dict(temporalLayer=2, layerNorm=True, dropout=0.3),
    "subsample_lstm_ln": dict(temporalLayer=2, cell="lstm", layerNorm=True, subsample=2, subsampleLayer=2),
    "subsample_relu_L1": dict(temporalLayer=2, subsample=3, subsampleLayer=1, dropout=0.2),
}


@pytest.mark.parametrize("name", list(GIVEN))
def test_back_propagation_through_given_activations_is_the_same(name):
    """costAndGradGiven on the net's own activations = costAndGrad, bit for bit (the GPU tests feed it the device's)."""
    kw = dict(GIVEN[name])
    np.random.seed(2)
    nn = Net(7, 5, 12, kw.pop("N", 4), 9, round_f32=False, **kw)
    nn.initParams()
    nn.dropoutStep, nn.utt = 2, 3
    data = np.random.RandomState(1).randn(7, 9)
    labels = np.array([1, 3, 2], dtype=np.int32)
    c1, g1, skip = nn.costAndGrad(data, labels)
    assert not skip
    g1 = [[a.copy(), b.copy()] for a, b in g1]
    h, temporal, _ = nn.forward(data)
    c2, g2, _ = nn.costAndGradGiven(data, labels, h[1:], temporal)
    assert c1 == c2
    for (a, b), (x, y) in zip(g1, g2):
        assert np.array_equal(a, x) and np.array_equal(b, y)


# ------------------------------------------------------------------------------------------- torch
@pytest.mark.parametrize("uni", [True, False])
def test_oracle_matches_torch_lstm(uni):
    """One LSTM layer of the oracle against torch.nn.LSTM in float64 (bias_hh = 0), per utterance of a ragged batch:
    the forward h of each direction, and the gradients of sum(out * R) w.r.t. the input, W_ih, b_ih and W_hh."""
    torch = pytest.importorskip("torch")
    rng = np.random.RandomState(5)
    n, H = 7, 6
    ndir = 1 if uni else 2
    lstm = torch.nn.LSTM(n, H, bidirectional=not uni).double()
    with torch.no_grad():
        for name, p in lstm.named_parameters():
            p.copy_(torch.from_numpy(rng.uniform(-0.6, 0.6, tuple(p.shape))))
            if name.startswith("bias_hh"):
                p.zero_()
    sfx = ["", "_reverse"][:ndir]
    W = np.concatenate([getattr(lstm, "weight_ih_l0" + s).detach().numpy() for s in sfx])
    b = np.concatenate([getattr(lstm, "bias_ih_l0" + s).detach().numpy() for s in sfx])
    Us = [getattr(lstm, "weight_hh_l0" + s).detach().numpy() for s in sfx]
    for T in (1, 2, 9, 5):      # the utterances of a ragged batch, each run at its own length
        x = rng.randn(n, T)
        Rw = rng.randn(H, T)
        xt = torch.from_numpy(x.T[:, None, :].copy()).requires_grad_(True)
        out, _ = lstm(xt)
        out = out[:, 0, :].T     # [ndir*H][T]
        loss = sum((out[d * H:(d + 1) * H] * torch.from_numpy(Rw)).sum() for d in range(ndir))
        loss.backward()
        pre = W.dot(x) + b[:, None]
        dz_all = []
        plain = (np.zeros((3, H)), np.zeros((H, T)), np.zeros((H, T)))     # no peepholes, no zoneout
        for d in range(ndir):
            gates, c, h = lstm_direction(pre[d * 4 * H:(d + 1) * 4 * H], Us[d], d == 1, *plain)
            np.testing.assert_allclose(h, out[d * H:(d + 1) * H].detach().numpy(), rtol=1e-12, atol=1e-13)
            dz, dU, _ = lstm_direction_bptt(Rw, gates, c, h, Us[d], d == 1, *plain)
            np.testing.assert_allclose(dU, getattr(lstm, "weight_hh_l0" + sfx[d]).grad.numpy(), rtol=1e-10, atol=1e-12)
            dz_all.append(dz)
        dz = np.concatenate(dz_all)
        np.testing.assert_allclose(dz.dot(x.T), np.concatenate([getattr(lstm, "weight_ih_l0" + s).grad.numpy()
                                                                for s in sfx]), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(dz.sum(axis=1), np.concatenate([getattr(lstm, "bias_ih_l0" + s).grad.numpy()
                                                                   for s in sfx]), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(W.T.dot(dz), xt.grad.numpy()[:, 0, :].T, rtol=1e-10, atol=1e-12)
        lstm.zero_grad()


def test_oracle_normalisation_is_torch_layer_norm():
    torch = pytest.importorskip("torch")
    rng = np.random.RandomState(1)
    for H, T, shift in ((13, 9, 0.0), (64, 5, 300.0), (7, 3, -2.0)):
        z = rng.randn(H, T) * rng.rand(1, T) * 3 + shift
        z[:, 0] = 0.25                               # a constant frame: var = 0
        gamma, beta = rng.randn(H, 1), rng.randn(H, 1)
        xh, rstd = layer_norm(z)
        ref = torch.nn.functional.layer_norm(torch.from_numpy(z.T.copy()), (H,), torch.from_numpy(gamma[:, 0].copy()),
                                             torch.from_numpy(beta[:, 0].copy()), eps=1e-5).numpy().T
        assert np.allclose(gamma * xh + beta, ref, rtol=1e-9, atol=1e-9)
        # and its backward against torch's autograd
        zt = torch.from_numpy(z.T.copy()).requires_grad_()
        gt = torch.from_numpy(gamma[:, 0].copy()).requires_grad_()
        bt = torch.from_numpy(beta[:, 0].copy()).requires_grad_()
        g = rng.randn(H, T)
        torch.nn.functional.layer_norm(zt, (H,), gt, bt, eps=1e-5).backward(torch.from_numpy(g.T.copy()))
        dz, dgamma, dbeta = layer_norm_backward(g, gamma, xh, rstd)
        assert np.allclose(dz, zt.grad.numpy().T, rtol=1e-10, atol=1e-10)
        assert np.allclose(dgamma[:, 0], gt.grad.numpy(), rtol=1e-10, atol=1e-12)
        assert np.allclose(dbeta[:, 0], bt.grad.numpy(), rtol=1e-10, atol=1e-12)


def _torch_net(o, datas, labels):
    """The same net as Net o (clipped-ReLU temporal layers, layer norm, dropout, subsampling; no LSTM) in torch float64
    with autograd and torch's CTC: (summed cost, gradient of every tensor)."""
    import torch
    P = [[torch.tensor(w, requires_grad=True), torch.tensor(b, requires_grad=True)] for w, b in o.stack]
    total = 0.0
    for u, (d, lab) in enumerate(zip(datas, labels)):
        o.utt = u
        x = torch.tensor(np.asarray(d, dtype=np.float64))
        for i in range(1, o.numLayers + 2):
            if o.stacked(i):
                n, T = x.shape
                Tp = frames(T, o.k)
                x = torch.cat([x, torch.zeros(n, Tp * o.k - T, dtype=x.dtype)], 1).T.reshape(Tp, o.k * n).T
            w, b = P[i - 1]
            z = w @ x + b
            T = z.shape[1]
            if o.temporal(i):
                idx = o.rec(i - o.temporalLayer)

                def sweep(U, order, prev):
                    cols = [None] * T
                    for m, t in enumerate(order):
                        v = z[:, t] + (U @ cols[t + prev] if m else 0.0)
                        cols[t] = torch.clamp(v, 0.0, o.maxAct)
                    return torch.stack(cols, 1)
                For = sweep(P[idx[0]][0], range(T), -1)
                z = For if o.unidirectional else For + sweep(P[idx[1]][0], range(T - 1, -1, -1), 1)
            elif i <= o.numLayers:
                if o.normed(i):
                    g, be = P[o.ln_index(i)]
                    z = torch.nn.functional.layer_norm(z.T, (z.shape[0],), g[:, 0], be[:, 0], eps=1e-5).T
                z = torch.relu(z)
                if o.dropped(i):
                    keep = o.drop(np.ones(tuple(z.shape)), i)
                    z = z * torch.tensor(keep)
            x = z
        lp = torch.log_softmax(x.T, 1)[:, None, :]
        total = total + torch.nn.functional.ctc_loss(lp, torch.tensor(lab, dtype=torch.long)[None],
                                                     torch.tensor([lp.shape[0]]), torch.tensor([len(lab)]),
                                                     blank=0, reduction="sum")
    total.backward()
    g = lambda t: np.zeros(tuple(t.shape)) if t.grad is None else t.grad.numpy()     # noqa: E731 (the dummies)
    return total.item(), [[g(w), g(b)] for w, b in P]


@pytest.mark.parametrize("name", [n for n in SUBSAMPLE if SUBSAMPLE[n][5].get("cell") != "lstm"])
def test_oracle_matches_torch_autograd(name):
    pytest.importorskip("torch")
    np.random.seed(7)
    kw = _subsampled(name, reg=0.0, round_f32=False)
    o = Net(*kw.pop("dims"), **kw)
    o.initParams()
    datas, labels = recipes.synth_batch(5, 6, LENS, NLABS, seed=3)
    costs, grad, skips = o.costAndGradBatch(datas, labels)
    assert not skips.any()
    tc, tg = _torch_net(o, datas, labels)
    assert abs(costs.sum() - tc) <= 1e-9 * abs(tc)
    for (a, b), (c, d) in zip(grad, tg):
        assert np.allclose(a, c, rtol=1e-8, atol=1e-11) and np.allclose(b, d, rtol=1e-8, atol=1e-11)


# ------------------------------------------------------------------------------------------- subsampling
def test_stack_and_unstack_follow_the_definition():
    rng = np.random.RandomState(0)
    for n, T, k in ((3, 7, 2), (5, 9, 3), (4, 2, 3), (1, 1, 4), (6, 12, 3)):
        x = rng.randn(n, T)
        S = stack_frames(x, k)
        assert S.shape == (k * n, frames(T, k))
        for tp in range(S.shape[1]):
            for m in range(k):
                t = k * tp + m
                assert np.array_equal(S[m * n:(m + 1) * n, tp], x[:, t] if t < T else np.zeros(n))
        assert np.array_equal(unstack_frames(S, k, T), x)


def test_utterance_too_short_for_its_labels_at_the_reduced_rate_is_skipped():
    """T = 7 frames, k = 3: 3 output frames, which 3 labels with a repeat cannot be aligned to: the CTC's own skip (the
    host rule for fewer frames than labels is test_admission_compares_ceil_t_over_k_with_the_labels)."""
    np.random.seed(1)
    o = Net(5, 6, 6, 3, 40, temporalLayer=2, subsample=3, subsampleLayer=1)
    o.initParams()
    cost, _, skip = o.costAndGrad(np.random.RandomState(0).randn(5, 7), np.array([1, 2, 2], dtype=np.int32))
    assert skip
