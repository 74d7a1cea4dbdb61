"""CPU tests of the peephole connections of the LSTM cell (ctcb_brnn_config.peephole = 1): the float64 restatement
(tests/net_oracle.py) with peepholes and P = 0 is its net without peepholes, bit for bit; with P drawn
non-zero it agrees with an independent torch-autograd restatement of the cell and with central differences on every
tensor; peephole = 0 answers
every config query as before; the config contract and the tensor table of peephole = 1; runNNet's flag."""
import ctypes
import os

import numpy as np
import pytest

import config_matrix
import recipes
from net_oracle import Net, lstm_direction, lstm_direction_bptt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _draw_p(net, seed, scale=0.5):
    """P of every direction of every LSTM layer uniform in (-scale, scale)."""
    rng = np.random.RandomState(seed)
    for j in range(net.numTemporal):
        for d in range(net.nrec):
            P = net.stack[net.peep_index(j, d)][0]
            P[...] = rng.uniform(-scale, scale, P.shape)


# ------------------------------------------------------------------------------------------- P = 0 is today's cell
@pytest.mark.parametrize("kw", [dict(temporalLayer=2), dict(temporalLayer=2, unidirectional=True),
                                dict(temporalLayer=1, numTemporal=2), dict(temporalLayer=1, numTemporal=2,
                                                                           unidirectional=True)],
                         ids=["bi", "uni", "stack2_bi", "stack2_uni"])
def test_zero_peepholes_are_the_cell_without_them(kw):
    """initParams draws the same numbers with and without peepholes and sets P = 0; the costs and every gradient of the
    shared tensors are then bit for bit those of the net without peepholes."""
    nets = []
    for peep in (False, True):
        np.random.seed(4)
        n = Net(7, 5, 6, 3, 9, cell="lstm", reg=1e-3, round_f32=False, peephole=peep, **kw)
        n.initParams()
        nets.append(n)
    off, on = nets
    base = len(off.stack)
    assert len(on.stack) == base + on.numTemporal * on.nrec
    for (w, b), (x, y) in zip(off.stack, on.stack):
        assert np.array_equal(w, x) and np.array_equal(b, y)
    assert all(not np.any(w) and w.shape == (3, 6) and b.shape == (1, 1) for w, b in on.stack[base:])
    datas, labels = recipes.synth_batch(7, 5, [9, 6, 4], [3, 2, 2], seed=2)
    c0, g0, s0 = off.costAndGradBatch(datas, labels)
    c1, g1, s1 = on.costAndGradBatch(datas, labels)
    assert np.array_equal(c0, c1) and np.array_equal(s0, s1) and off.regcost == on.regcost
    for (a, b), (x, y) in zip(g0, g1):
        assert np.array_equal(a, x) and np.array_equal(b, y)
    assert all(np.any(w) and not np.any(b) for w, b in g1[base:])     # dP is not trivially 0, the dummies are


# ------------------------------------------------------------------------------------------- against torch
def _torch_peephole_direction(pre, U, P, reverse, R):
    """The peephole cell of one direction in torch float64, written from its definition: returns h [H][T] and the
    gradients of sum(h * R) w.r.t. pre, U and P."""
    import torch
    pre_t = torch.tensor(pre, requires_grad=True)
    U_t = torch.tensor(U, requires_grad=True)
    P_t = torch.tensor(P, requires_grad=True)
    H, T = U.shape[1], pre.shape[1]
    h = torch.zeros(H, dtype=torch.float64)
    c = torch.zeros(H, dtype=torch.float64)
    hs = [None] * T
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        z = pre_t[:, t] + U_t @ h
        i = torch.sigmoid(z[:H] + P_t[0] * c)
        f = torch.sigmoid(z[H:2 * H] + P_t[1] * c)
        g = torch.tanh(z[2 * H:3 * H])
        c = f * c + i * g
        o = torch.sigmoid(z[3 * H:] + P_t[2] * c)
        h = o * torch.tanh(c)
        hs[t] = h
    hh = torch.stack(hs, 1)
    (hh * torch.tensor(R)).sum().backward()
    return hh.detach().numpy(), pre_t.grad.numpy(), U_t.grad.numpy(), P_t.grad.numpy()


@pytest.mark.parametrize("reverse", [False, True])
def test_oracle_cell_matches_torch_autograd(reverse):
    """The oracle's forward and hand-written BPTT of one direction against autograd of the cell's definition, for the
    utterances of a ragged batch (T = 1 included)."""
    pytest.importorskip("torch")
    rng = np.random.RandomState(9)
    H = 5
    for T in (1, 2, 7, 4):
        pre = rng.uniform(-1.5, 1.5, (4 * H, T))
        U = rng.uniform(-0.6, 0.6, (4 * H, H))
        P = rng.uniform(-0.5, 0.5, (3, H))
        R = rng.randn(H, T)
        h_t, dpre, dU_t, dP_t = _torch_peephole_direction(pre, U, P, reverse, R)
        zero = np.zeros((H, T))     # no zoneout
        gates, c, h = lstm_direction(pre, U, reverse, P, zero, zero)
        np.testing.assert_allclose(h, h_t, rtol=1e-12, atol=1e-14)
        dz, dU, dP = lstm_direction_bptt(R, gates, c, h, U, reverse, P, zero, zero)
        np.testing.assert_allclose(dz, dpre, rtol=1e-10, atol=1e-13)
        np.testing.assert_allclose(dU, dU_t, rtol=1e-10, atol=1e-13)
        np.testing.assert_allclose(dP, dP_t, rtol=1e-10, atol=1e-13)
        assert T == 1 or np.abs(dP[:2]).max() > 1e-3      # the i and f peepholes take part


# ------------------------------------------------------------------------------------------- central differences
def _probe(x, idx, cost):
    eps = 1e-6
    old = x[idx]
    x[idx] = old + eps
    cp = cost()
    x[idx] = old - eps
    cm = cost()
    x[idx] = old
    return (cp - cm) / (2 * eps)


# name: Net arguments (dims = inputDim, outputDim, layerSize, numLayers, maxBatch), lengths
FD = {
    "bi": (dict(dims=(5, 6, 4, 3, 7), temporalLayer=2), [7, 7]),
    "uni": (dict(dims=(5, 6, 4, 3, 7), temporalLayer=2, unidirectional=True), [7, 7]),
    "stack2": (dict(dims=(5, 6, 4, 4, 7), temporalLayer=2, numTemporal=2), [7, 7]),
    "ragged": (dict(dims=(5, 6, 4, 3, 9), temporalLayer=1, numTemporal=2, unidirectional=True), [9, 4, 6]),
    "layernorm": (dict(dims=(5, 6, 6, 3, 8), temporalLayer=2, layerNorm=True), [8, 5]),
    "dropout": (dict(dims=(5, 6, 6, 4, 8), temporalLayer=2, dropout=0.3, dropoutSeed=5), [8, 5]),
    "subsample_below": (dict(dims=(5, 6, 6, 3, 13), temporalLayer=2, subsample=2, subsampleLayer=1), [13, 8, 11]),
    "subsample_above": (dict(dims=(5, 6, 6, 3, 13), temporalLayer=1, subsample=3, subsampleLayer=2), [13, 8, 11]),
}


@pytest.mark.parametrize("name", list(FD))
def test_oracle_gradient_matches_central_differences(name):
    """P drawn non-zero, reg > 0, weights twice the initial scale, biases off 0: 3 entries of every tensor (every entry
    of every P) against the central difference of the summed cost, |analytic - numeric| <= 1e-6 max(1, |numeric|)."""
    kw, lens = dict(FD[name][0]), FD[name][1]
    net = Net(*kw.pop("dims"), reg=1e-3, round_f32=False, cell="lstm", peephole=True, **kw)
    np.random.seed(11)
    net.initParams()
    for w, _ in net.stack:
        w *= 2.0
    for _, b in net.stack[:net.numLayers + 1]:      # off 0: a frame whose input is all dropped would sit on the kink
        b += 0.1 * np.random.RandomState(4).randn(*b.shape)
    _draw_p(net, 3)
    if net.dropout:
        net.dropoutStep = 2
    datas, labels = recipes.synth_batch(net.inputDim, net.outputDim, lens, [2] * len(lens), seed=3)
    _, grad, skips = net.costAndGradBatch(datas, labels)
    assert not skips.any()
    peeps = {net.peep_index(j, d) for j in range(net.numTemporal) for d in range(net.nrec)}
    dummies = set(range(net.numLayers + 1, net.numLayers + 1 + net.numTemporal * net.nrec)) | peeps
    f = lambda: net.costAndGradBatch(datas, labels)[0].sum() + net.regcost        # noqa: E731
    rng = np.random.RandomState(2)
    for ti, (w, b) in enumerate(net.stack):
        for x, gx in ((w, grad[ti][0]), (b, grad[ti][1])):
            if ti in dummies and x is b:
                assert not np.any(gx)
                continue
            idxs = list(np.ndindex(x.shape)) if ti in peeps else \
                [tuple(rng.randint(0, s) for s in x.shape) for _ in range(3)]
            for idx in idxs:
                num = _probe(x, idx, f)
                assert abs(num - gx[idx]) <= 1e-6 * max(1.0, abs(num)), (ti, idx, num, gx[idx])
    assert all(np.abs(grad[t][0][:2]).max() > 1e-4 and np.abs(grad[t][0][2]).max() > 1e-4 for t in peeps)


def test_back_propagation_through_given_activations_is_the_same():
    """costAndGradGiven on the net's own activations = costAndGrad, bit for bit, with non-zero P."""
    np.random.seed(2)
    nn = Net(7, 5, 12, 4, 9, temporalLayer=2, numTemporal=2, cell="lstm", peephole=True, round_f32=False)
    nn.initParams()
    _draw_p(nn, 4)
    data = np.random.RandomState(1).randn(7, 9)
    labels = np.array([1, 3, 2], dtype=np.int32)
    c1, g1, _ = nn.costAndGrad(data, labels)
    g1 = [[a.copy(), b.copy()] for a, b in g1]
    h, temporal, _ = nn.forward(data)
    c2, g2, _ = nn.costAndGradGiven(data, labels, h[1:], temporal)
    assert c1 == c2
    for (a, b), (x, y) in zip(g1, g2):
        assert np.array_equal(a, x) and np.array_equal(b, y)


def test_oracle_refuses_peepholes_without_the_lstm_cell():
    with pytest.raises(ValueError, match="peephole.*cell='lstm'.*'relu'"):
        Net(7, 5, 6, 3, 9, temporalLayer=2, peephole=True)


# ------------------------------------------------------------------------------------------- the config contract
def _cfg(D, K, H, N, tl, T, B, uni=0, nt=1, cell=1, ln=0, k=0, sl=0, peep=1):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, T, B, 9, 0.0, 20.0, uni, nt, cell, ln, k, sl, peep)


def _table(cfg):
    from _ctcb import lib
    n = lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for i in range(n):
        assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        out.append((off.value, r.value, c.value))
    return out


def _golden():
    """The fixture of the machine the library plans for: no device, or an H100 SXM (sm_90, 132 SMs); None for any
    other device."""
    import torch
    if not torch.cuda.is_available():
        return os.path.join(GOLDEN, "subsample_configs.npz")
    p = torch.cuda.get_device_properties(0)
    if (p.major, p.minor, p.multi_processor_count) == (9, 0, 132):
        return os.path.join(GOLDEN, "subsample_configs_h100_sxm.npz")
    return None


def test_peepholes_off_answer_every_config_query_as_before():
    """peephole = 0 gives, for every config of the matrix, the answers of the build before the member existed (the
    fixtures of the subsampling change: one for a machine without a device, one for an H100 SXM)."""
    import _ctcb
    from _ctcb import lib
    golden = _golden()
    if golden is None:
        pytest.skip("the fixtures are those of no device and of an H100 SXM (sm_90, 132 SMs), not of this device")
    want = np.load(golden)["digests"]
    config_matrix.bind(lib, _ctcb.BrnnConfig)
    got = []
    for e in config_matrix.MATRIX:
        cfg = config_matrix.config(_ctcb.BrnnConfig, e)
        cfg.peephole = 0
        got.append(config_matrix.digest(config_matrix.answers(lib, cfg)))
    bad = np.nonzero(np.array(got, dtype=np.int64) != want)[0]
    assert len(bad) == 0, [config_matrix.MATRIX[i] for i in bad[:5]]


def test_invalid_peepholes_are_refused_with_a_message():
    from _ctcb import lib
    h = ctypes.c_void_p()
    for cell, peep, text in ((0, 1, "peephole 1 needs the LSTM cell (cell 1); cell is 0"),
                             (1, 2, "peephole 2 is neither 0 (off) nor 1"), (1, -1, "peephole -1 is neither")):
        cfg = _cfg(13, 11, 64, 3, 2, 60, 8, cell=cell, peep=peep)
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
        assert text in lib.ctcb_last_error().decode(), lib.ctcb_last_error()
        assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_num_tensors(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == 0


def test_peephole_layout_over_the_config_matrix():
    """For every valid LSTM config of the matrix (and subsampled ones): every tensor of the net without peepholes keeps
    its offset and shape, the [P (3 x H), dummy] entries follow in the recurrent entries' order, the early all-reduce
    range (W of the lowest temporal layer to the end of b of the last map) is unchanged, the forward workspace and its
    flag offset are unchanged, the training workspace is never smaller and every activation offset is unchanged.
    Without a temporal layer nothing changes at all."""
    import _ctcb
    from _ctcb import lib
    n = 0
    f0, f1 = ctypes.c_size_t(), ctypes.c_size_t()
    o0, o1, w0, w1 = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int32(), ctypes.c_int32()
    for e in config_matrix.MATRIX:
        if e[7] != 1:
            continue
        for k, sl in ((0, 0), (2, 1), (3, 3)):
            off = config_matrix.config(_ctcb.BrnnConfig, e, k, sl)
            on = config_matrix.config(_ctcb.BrnnConfig, e, k, sl)
            on.peephole = 1
            a, b = _table(off), _table(on)
            if not a:
                assert not b
                continue
            n += 1
            D, K, H, N, tl, nt, uni = e[:7]
            ntemp = (max(1, nt) if 0 < tl <= N else 0)
            extra = ntemp * (1 if uni else 2)
            assert len(b) == len(a) + 2 * extra and b[:len(a)] == a
            end = a[-1][0] + a[-1][1] * a[-1][2]
            for x in range(extra):
                assert b[len(a) + 2 * x][1:] == (3, H) and b[len(a) + 2 * x + 1][1:] == (1, 1)
                assert b[len(a) + 2 * x][0] >= end
                end = b[len(a) + 2 * x + 1][0] + 1
            if ntemp:       # the early range is read from tensors that did not move
                lo, hi = b[2 * tl][0], b[2 * N + 1][0] + K
                assert (lo, hi) == (a[2 * tl][0], a[2 * N + 1][0] + K) and hi <= a[-1][0] + 1
            p0, p1 = lib.ctcb_brnn_param_count(ctypes.byref(off)), lib.ctcb_brnn_param_count(ctypes.byref(on))
            assert p1 == (p0 if not extra else (end + 3) // 4 * 4)
            t0, t1 = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off)), lib.ctcb_brnn_workspace_bytes(ctypes.byref(on))
            assert t1 >= t0 and (t1 == t0) == (extra == 0)
            flag = lib.ctcb_brnn_error_flag_offset
            assert flag(ctypes.byref(on)) == flag(ctypes.byref(off))
            assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), ctypes.byref(f0)) == \
                lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(on), ctypes.byref(f1)) and f0.value == f1.value
            for what in (0, 1, 3, 4, 5, 6):
                for layer in range(N + 2):
                    r0 = lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, layer, ctypes.byref(o0),
                                                         ctypes.byref(w0))
                    r1 = lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, layer, ctypes.byref(o1),
                                                         ctypes.byref(w1))
                    assert r0 == r1 and (r0 or (o0.value, w0.value) == (o1.value, w1.value))
    assert n > 1000


def test_peephole_partials_go_behind_everything_else():
    """C3-like bi-directional LSTM layer (1024 units, 800 x 128 frames): the training workspace grows by exactly the
    partial sums of the peephole gradients, ceil(102400 / 1024) chunks of 2 x 3 x 1024 floats."""
    from _ctcb import lib
    al = lambda x: (x + 255) // 256 * 256     # noqa: E731
    off, on = _cfg(41, 32, 1024, 3, 2, 800, 128, peep=0), _cfg(41, 32, 1024, 3, 2, 800, 128)
    grow = lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) - lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    assert grow == al(100 * 6 * 1024 * 4) == lib.ctcb_lstm_peephole_grad_workspace_bytes(800, 128, 1024, 2)
    # above a subsampling point at k = 2: the lowest LSTM layer has 400 x 128 frames
    off, on = _cfg(41, 32, 1024, 3, 2, 800, 128, k=2, sl=1, peep=0), _cfg(41, 32, 1024, 3, 2, 800, 128, k=2, sl=1)
    grow = lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) - lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    assert grow == al(50 * 6 * 1024 * 4)


def test_entry_points_check_their_arguments():
    from _ctcb import lib
    assert lib.ctcb_lstm_peephole_grad_workspace_bytes(4, 2, 8, 3) == 0
    assert lib.ctcb_lstm_peephole_grad_f32(4, 2, 8, None, None, None, None, None, 0, None, 0, None) == -1
    assert "null pointer" in lib.ctcb_last_error().decode()
    assert lib.ctcb_lstm_sweep_peephole_f32(0, 4, 2, 8, None, None, None, None, None, None, None, None, None, None,
                                            None, None, None, 0, None) == -1
    assert "ctcb_lstm_sweep_peephole_f32: null pointer" in lib.ctcb_last_error().decode()


# ------------------------------------------------------------------------------------------- runNNet
def test_runnnet_peephole_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).peephole is False
    o = runNNet._parse(["--cell", "lstm", "--peephole"])
    assert o.peephole is True
    cfg = runNNet.run_config(o)
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.trained_config(f).peephole is True                                      # --test rebuilds it
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["peephole"] is True       # resume keeps it
    old = dict(cfg)
    del old["peephole"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.trained_config(f2).peephole is False                                    # a model from before
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["peephole"] is False
