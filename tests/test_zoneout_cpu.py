"""CPU tests of zoneout on the LSTM cell: the mask restatement (tests/net_oracle.py) against a plain loop, its keep
rates, its counters against the other draws of a seed, the float64 cell against a torch-autograd restatement and
against central differences, and the C ABI's config, setter, workspace and runNNet contract (no device work)."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from net_oracle import Net, lstm_direction, lstm_direction_bptt, philox4x32_10, zoneout_masks, zoneout_threshold


def _loop_masks(zc, zh, seed, step, layer, d, g, T, H):
    """The rule of include/ctcb200.h one unit at a time, from the Philox blocks alone."""
    lc, lh = np.zeros((T, H), bool), np.zeros((T, H), bool)
    tc = int(np.floor(float(np.float32(zc)) * 2.0 ** 32))
    th = int(np.floor(float(np.float32(zh)) * 2.0 ** 32))
    for t in range(T):
        for j in range(H):
            ctr = np.array([[step % 2 ** 32, g % 2 ** 32, t, (layer << 24) | (d << 23) | j]], dtype=np.uint64)
            r = [int(x) for x in philox4x32_10(ctr, (seed % 2 ** 32, seed >> 32))[0]]
            lc[t, j], lh[t, j] = r[0] < tc, r[1] < th
    return lc, lh


@pytest.mark.parametrize("case", [
    (0.1, 0.05, 33, 0, 2, 0, 0, 7, 9),
    (0.5, 0.9, 2 ** 40 + 5, 2 ** 33 + 7, 1, 1, 2 ** 32 + 3, 5, 4),       # step and g wrap at 2^32
    (0.999, 0.0, 2 ** 64 - 1, 12, 64, 1, 11, 3, 70),
])
def test_restatement_equals_a_plain_loop(case):
    zc, zh, seed, step, layer, d, g, T, H = case
    lc, lh = zoneout_masks(zc, zh, seed, step, layer, d, g, T, H)
    wc, wh = _loop_masks(zc, zh, seed, step, layer, d, g, T, H)
    assert np.array_equal(lc, wc) and np.array_equal(lh, wh)


@pytest.mark.parametrize("z", [0.05, 0.15, 0.5, 0.9])
def test_keep_rates_follow_their_binomial_law(z):
    """The kept count of 200 x 256 units is Binomial(n, floor(z 2^32) / 2^32): a two-sided 1e-6 test, per word."""
    lc, lh = zoneout_masks(z, z, 7, 3, 2, 1, 5, 200, 256)
    p = zoneout_threshold(z) / 2.0 ** 32
    for m in (lc, lh):
        assert stats.binomtest(int(m.sum()), m.size, p).pvalue > 1e-6
    assert 0.0 < np.mean(lc != lh) < 1.0 or z == 0.0        # the two words are separate draws
    lc0, lh0 = zoneout_masks(0.0, 0.0, 7, 3, 2, 1, 5, 50, 64)
    assert not lc0.any() and not lh0.any()


def test_counters_never_meet_dropout_input_masks_or_weight_noise():
    """Zoneout's fourth word is (i << 24) | (d << 23) | j with i a temporal layer's index >= 1; dropout's is
    (i' << 24) | q with i' a non-temporal layer's index, so the top 8 bits differ; SpecAugment's is < 2^24 (third
    word 0); weight noise's third word is 1 and its fourth 0.  Checked on sampled counters of each, every layer of a
    net with temporal layers 2..3 of 5."""
    steps, gs, ts = [0, 1, 2 ** 32 - 1, 2 ** 40 + 3], [0, 1, 5], [0, 1, 2, 70]
    temporal, hidden = (2, 3), (1, 4, 5)
    ours = [(s & 0xFFFFFFFF, g, t, (i << 24) | (d << 23) | j) for s in steps for g in gs for t in ts
            for i in temporal for d in (0, 1) for j in (0, 1, 255, 2 ** 23 - 1)]
    drop = [(s & 0xFFFFFFFF, g, t, (i << 24) | q) for s in steps for g in gs for t in ts for i in hidden
            for q in (0, 1, 63, 2 ** 22)]
    masks = [(s & 0xFFFFFFFF, g, 0, k) for s in steps for g in gs for k in (0, 1, 127, 2 ** 24 - 1)]
    noise = [(s & 0xFFFFFFFF, q, 1, 0) for s in steps for q in (0, 1, 2, 5, 2 ** 32 - 1)]
    o = set(ours)
    assert all(c[3] >= 2 ** 24 for c in ours) and all(c[3] < 2 ** 24 for c in masks)
    assert not o & set(drop) and not o & set(masks) and not o & set(noise)


# ------------------------------------------------------------------------------------------------ the float64 net
D, K = 7, 5
NETS = {
    "bi_k1": dict(temporalLayer=2, numTemporal=1),
    "uni_k2": dict(temporalLayer=1, numTemporal=2, unidirectional=True),
    "bi_k2_ln_drop_sub": dict(temporalLayer=2, numTemporal=2, layerNorm=True, dropout=0.3, subsample=2,
                              subsampleLayer=2),
}


def _data(T=9, seed=3, L=3):
    rng = np.random.RandomState(seed)
    return rng.randn(D, T).astype(np.float32).astype(np.float64), rng.randint(1, K, size=L).astype(np.int32)


def _net(name, peephole, round_f32=True, **z):
    kw = dict(NETS[name], cell="lstm", reg=1e-3, dropoutSeed=5, round_f32=round_f32)
    np.random.seed(4)
    net = Net(D, K, 6, 4, 20, peephole=peephole, **kw, **z)
    net.initParams()
    if peephole:
        rng = np.random.RandomState(8)
        for k in range(len(net.stack) - net.entries(), len(net.stack), 2):
            net.stack[k][0][...] = rng.uniform(-0.5, 0.5, net.stack[k][0].shape)
    net.dropoutStep, net.utt = 2, 1
    return net


def _torch_direction(P, U, reverse, peep, lc, lh):
    """The zoneout cell in torch, for autograd: the forward of include/ctcb200.h spelt out."""
    H = U.shape[1]
    T = P.shape[1]
    hp = torch.zeros(H, dtype=P.dtype)
    cp = torch.zeros(H, dtype=P.dtype)
    hs = [None] * T
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        z = P[:, t] + U @ hp
        zi, zf, zg, zo_ = z[:H], z[H:2 * H], z[2 * H:3 * H], z[3 * H:]
        if peep is not None:
            zi, zf = zi + peep[0] * cp, zf + peep[1] * cp
        ct = torch.sigmoid(zf) * cp + torch.sigmoid(zi) * torch.tanh(zg)
        cp = lc[:, t] * cp + (1 - lc[:, t]) * ct
        if peep is not None:
            zo_ = zo_ + peep[2] * cp
        hp = lh[:, t] * hp + (1 - lh[:, t]) * torch.sigmoid(zo_) * torch.tanh(cp)
        hs[t] = hp
    return torch.stack(hs, dim=1)


@pytest.mark.parametrize("mode", ["masks", "expectation"])
@pytest.mark.parametrize("peephole", [False, True])
@pytest.mark.parametrize("reverse", [False, True])
def test_cell_matches_torch_autograd_and_central_differences(mode, peephole, reverse):
    """One direction: dz, dU and dP of the oracle's BPTT against autograd of the torch cell (pre-activations P, U, the
    peepholes), and dP, dU against central differences of sum(w * h)."""
    H, T = 5, 11
    rng = np.random.RandomState(11)
    P = rng.randn(4 * H, T)
    U = rng.uniform(-0.6, 0.6, (4 * H, H))
    peep = rng.uniform(-0.5, 0.5, (3, H)) if peephole else None
    p64 = peep if peephole else np.zeros((3, H))     # the oracle's cell without peepholes: P = 0
    if mode == "masks":
        lc, lh = zoneout_masks(0.4, 0.3, 9, 1, 2, int(reverse), 3, T, H)
        lc, lh = lc.T.astype(np.float64), lh.T.astype(np.float64)
        assert lc.any() and lh.any() and not lc.all() and not lh.all()
    else:
        lc, lh = np.full((H, T), 0.4), np.full((H, T), 0.3)
    w = rng.randn(H, T)
    gates, c, h = lstm_direction(P, U, reverse, p64, lc, lh)
    dz, dU, dP = lstm_direction_bptt(w, gates, c, h, U, reverse, p64, lc, lh)
    tP, tU = torch.tensor(P, requires_grad=True), torch.tensor(U, requires_grad=True)
    tpeep = torch.tensor(peep, requires_grad=True) if peephole else None
    th = _torch_direction(tP, tU, reverse, tpeep, torch.tensor(lc), torch.tensor(lh))
    assert np.allclose(th.detach().numpy(), h, rtol=1e-12, atol=1e-14)
    (th * torch.tensor(w)).sum().backward()
    assert np.allclose(tP.grad.numpy(), dz, rtol=1e-9, atol=1e-12)
    assert np.allclose(tU.grad.numpy(), dU, rtol=1e-9, atol=1e-12)
    if peephole:
        assert np.allclose(tpeep.grad.numpy(), dP, rtol=1e-9, atol=1e-12)

    def loss(P_, U_, peep_):
        return float(np.sum(w * lstm_direction(P_, U_, reverse, peep_, lc, lh)[2]))
    eps = 1e-6
    for arr, grad in ((P, dz), (U, dU)) + (((peep, dP),) if peephole else ()):
        for idx in [(0, 0), (arr.shape[0] - 1, arr.shape[1] - 1), (arr.shape[0] // 2, 1)]:
            old = arr[idx]
            arr[idx] = old + eps
            up = loss(P, U, p64)
            arr[idx] = old - eps
            dn = loss(P, U, p64)
            arr[idx] = old
            assert abs((up - dn) / (2 * eps) - grad[idx]) <= 1e-6 * max(1.0, abs(grad[idx]))


@pytest.mark.parametrize("peephole", [False, True])
def test_elementwise_check_accepts_the_rounded_oracle_and_rejects_a_flipped_lambda(peephole):
    """_check_forward / _check_bptt of test_lstm_plans_gpu.py with lambdas, the bounds the GPU's zoneout sweep is held
    to: net_oracle.lstm_direction's gates, c, h and its BPTT's dz, each rounded to float32, meet C_FWD and C_BPTT; the
    same arrays checked with one lambda_c, or one lambda_h, flipped at a frame where that changes c or h exceed them."""
    from test_lstm_plans_gpu import C_BPTT, C_FWD, _check_bptt, _check_forward
    H, T, B, nd = 6, 7, 3, 2
    rng = np.random.RandomState(5 + peephole)
    lens = np.array([T, 4, 1], np.int32)
    f32 = lambda a: np.asarray(a, np.float32)           # noqa: E731
    pre = f32(rng.uniform(-1.5, 1.5, (T, B, nd * 4 * H)))
    Us = [f32(rng.uniform(-0.8, 0.8, (4 * H, H))) for _ in range(nd)]
    Ps = [f32(rng.uniform(-0.5, 0.5, (3, H))) for _ in range(nd)] if peephole else None
    dh = f32(rng.randn(T, B, H))
    lc = [np.zeros((T, B, H)) for _ in range(nd)]
    lh = [np.zeros((T, B, H)) for _ in range(nd)]
    r = dict(gates=np.zeros((T, B, nd * 4 * H), np.float32), c=[np.zeros((T, B, H), np.float32) for _ in range(nd)],
             h=[np.zeros((T, B, H), np.float32) for _ in range(nd)], dz=np.zeros((T, B, nd * 4 * H), np.float32))
    for d in range(nd):
        blk = slice(d * 4 * H, (d + 1) * 4 * H)
        p64 = Ps[d].astype(np.float64) if peephole else np.zeros((3, H))
        for u, Tu in enumerate(lens):
            a, b = zoneout_masks(0.4, 0.3, 9, 1, 2, d, u, Tu, H)
            lc[d][:Tu, u], lh[d][:Tu, u] = a, b
            P = pre[:Tu, u, blk].T.astype(np.float64)
            g, c, h = lstm_direction(P, Us[d].astype(np.float64), d == 1, p64, lc[d][:Tu, u].T, lh[d][:Tu, u].T)
            dz = lstm_direction_bptt(dh[:Tu, u].T.astype(np.float64), g, c, h, Us[d].astype(np.float64), d == 1, p64,
                                     lc[d][:Tu, u].T, lh[d][:Tu, u].T)[0]
            r["gates"][:Tu, u, blk], r["c"][d][:Tu, u], r["h"][d][:Tu, u] = f32(g.T), f32(c.T), f32(h.T)
            r["dz"][:Tu, u, blk] = f32(dz.T)

    class Problem:
        pass
    sw = Problem()
    sw.H, sw.T, sw.B, sw.ndir, sw.lens, sw.pre, sw.Us, sw.Ps, sw.dh = H, T, B, nd, lens, pre, Us, Ps, dh
    fwd, dz = _check_forward(r, sw, lc, lh), _check_bptt(r, sw, lc, lh)
    assert fwd["gates"] <= C_FWD and fwd["c"] <= C_FWD and fwd["h"] <= C_FWD and fwd["kept"], fwd
    assert dz <= C_BPTT, dz
    # a frame of utterance 0, direction 0, where the new c (h) is far from the one it would keep
    c0, h0 = r["c"][0][:, 0].astype(np.float64), r["h"][0][:, 0].astype(np.float64)
    for lam, x, key in ((lc, c0, "c"), (lh, h0, "h")):
        gap = np.abs(x[2:] - x[1:-1])
        t, j = np.unravel_index(int(np.argmax(gap)), gap.shape)
        t += 2
        flipped = [a.copy() for a in lam]
        flipped[0][t, 0, j] = 1.0 - flipped[0][t, 0, j]
        args = (flipped, lh) if key == "c" else (lc, flipped)
        assert _check_forward(r, sw, *args)[key] > 10 * C_FWD, key
        assert _check_bptt(r, sw, *args) > C_BPTT, key


def test_whole_net_central_differences():
    """The net's gradient (masks drawn, peepholes, two stacked layers) against central differences of its cost on
    every tensor."""
    net = _net("bi_k2_ln_drop_sub", True, round_f32=False, zoneoutCell=0.3, zoneoutHidden=0.2)
    data, labels = _data()
    cost, grad, skip = net.costAndGrad(data, labels)
    assert not skip
    eps = 1e-6
    for k, (w, b) in enumerate(net.stack):
        for arr, g in ((w, grad[k][0]), (b, grad[k][1])):
            if arr.shape == (1, 1):
                continue
            idx = tuple(s // 2 for s in arr.shape)
            old = arr[idx]
            arr[idx] = old + eps
            up = net.costAndGrad(data, labels)[0]
            arr[idx] = old - eps
            dn = net.costAndGrad(data, labels)[0]
            arr[idx] = old
            assert abs((up - dn) / (2 * eps) - g[idx]) <= 1e-5 * max(1.0, abs(g[idx])), (k, idx)


def test_oracle_refuses_what_nnet_refuses():
    for bad in (-0.1, 1.0, float("nan")):
        with pytest.raises(ValueError):
            Net(D, K, 6, 3, 20, temporalLayer=2, cell="lstm", zoneoutCell=bad)
        with pytest.raises(ValueError):
            Net(D, K, 6, 3, 20, temporalLayer=2, cell="lstm", zoneoutHidden=bad)
    with pytest.raises(ValueError):
        Net(D, K, 6, 3, 20, temporalLayer=2, cell="relu", zoneoutCell=0.1)


# ------------------------------------------------------------------------------------------------------- C ABI
def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1, 1)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


CFG_CASES = {
    "bi_lstm": dict(),
    "uni_k2": dict(unidirectional=1, temporalLayer=1, numTemporal=2),
    "peephole_ln": dict(peephole=1, layerNorm=1),
    "subsample": dict(subsample=2, subsampleLayer=2, layerSize=63),
    "masks_noise": dict(maskFeatDim=41, weightNoise=1),
}


@pytest.mark.parametrize("name", list(CFG_CASES))
def test_workspace_grows_by_exactly_the_dh_carry(name):
    from _ctcb import lib
    off = _cfg(**CFG_CASES[name])
    assert off.zoneout == 0              # an initialiser without the member keeps its meaning
    on = _cfg(zoneout=1, **CFG_CASES[name])
    base = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    assert base > 0
    H, B = on.layerSize, on.maxB
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) == base + (2 * B * H * 4 + 255) // 256 * 256
    assert lib.ctcb_brnn_param_count(ctypes.byref(on)) == lib.ctcb_brnn_param_count(ctypes.byref(off))
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(on)) == lib.ctcb_brnn_num_tensors(ctypes.byref(off))
    assert (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(on), None)
            == lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), None))
    assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(on)) == lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))
    for what in range(7):
        for layer in range(5):
            a, b = ctypes.c_size_t(), ctypes.c_size_t()
            ra = lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, layer, ctypes.byref(a), None)
            rb = lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, layer, ctypes.byref(b), None)
            assert ra == rb and a.value == b.value, (what, layer)


def test_standalone_workspace_size():
    from _ctcb import lib
    for H, B in ((64, 8), (70, 5), (1024, 3)):
        carry = (2 * B * H * 4 + 255) // 256 * 256
        assert lib.ctcb_lstm_sweep_workspace_bytes(H, B) == 4096 + carry
        assert lib.ctcb_lstm_sweep_zoneout_workspace_bytes(H, B) == 4096 + 2 * carry
    assert lib.ctcb_lstm_sweep_zoneout_workspace_bytes(0, 3) == 0


def test_config_refusals():
    from _ctcb import lib
    for kw, text in ((dict(zoneout=2), b"zoneout 2"), (dict(zoneout=-1), b"zoneout -1"),
                     (dict(zoneout=1, cell=0), b"needs the LSTM cell")):
        cfg = _cfg(**kw)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, kw
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, kw
        assert text in lib.ctcb_last_error(), lib.ctcb_last_error()


def test_set_zoneout_argument_contract():
    from _ctcb import lib
    step = ctypes.c_int64(0)     # the setter only stores the pointer: a host address does for the contract
    sp = ctypes.addressof(step)
    h, h0 = ctypes.c_void_p(), ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg(zoneout=1)), ctypes.byref(h)) == 0
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg()), ctypes.byref(h0)) == 0
    n0 = lib.ctcb_launch_count()
    try:
        set_ = lib.ctcb_brnn_set_zoneout
        assert set_(h, 0.1, 0.05, 33, sp) == 0
        assert set_(h, 0.999, 0.0, 2 ** 64 - 1, sp) == 0
        assert set_(h, 0.2, 0.2, 1, None) == 0                  # a null step is for forward-only use
        assert set_(h, 0.0, 0.0, 0, None) == 0
        for bad in (-0.1, 1.0, 1.5, float("nan"), float("inf")):
            for args in ((bad, 0.0), (0.0, bad)):
                assert set_(h, *args, 1, sp) == -1, args
                msg = lib.ctcb_last_error()
                assert b"ctcb_brnn_set_zoneout" in msg and b"[0, 1)" in msg, msg
        assert set_(h0, 0.1, 0.0, 1, sp) == -1 and b"zoneout = 1" in lib.ctcb_last_error()
        assert set_(h0, 0.0, 0.1, 1, sp) == -1 and b"zoneout = 1" in lib.ctcb_last_error()
        assert set_(h0, 0.0, 0.0, 1, None) == 0
        assert set_(None, 0.0, 0.0, 1, sp) == -1 and b"null handle" in lib.ctcb_last_error()
        # a training call with z > 0 and no step counter is refused before it launches anything
        assert set_(h, 0.2, 0.1, 1, None) == 0
        cfg = _cfg(zoneout=1)
        ws = 1 << 20
        x = 1 << 24
        rc = lib.ctcb_brnn_cost_and_grad(h, x, x, x, x, 2, 10, x, x, x, x, None, None, None,
                                         ws, lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)), None)
        assert rc == -1 and b"step counter" in lib.ctcb_last_error(), lib.ctcb_last_error()
        # the sweep alone refuses its arguments before any device work
        f = lib.ctcb_lstm_sweep_zoneout_f32
        n = lib.ctcb_lstm_sweep_zoneout_workspace_bytes(64, 2)

        def sweep(zc=0.1, zh=0.1, train=1, step_=sp, first=0, stride=1, layer=1):
            return f(0, 4, 2, 64, x, x, x, x, None, None, x, x, x, x, None, None, zc, zh, train, 1, step_, first,
                     stride, layer, ws, n, None)
        for kw in (dict(zc=1.0), dict(zh=-0.5), dict(zc=float("nan")), dict(step_=None), dict(first=-1),
                   dict(stride=0), dict(layer=0), dict(layer=256)):
            assert sweep(**kw) == -1, kw
            assert b"ctcb_lstm_sweep_zoneout_f32" in lib.ctcb_last_error()
    finally:
        lib.ctcb_brnn_destroy(h)
        lib.ctcb_brnn_destroy(h0)
    assert lib.ctcb_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_zoneout_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    opts = runNNet._parse([])
    assert opts.zoneoutCell == 0.0 and opts.zoneoutHidden == 0.0
    assert all(any(f[0] == n and f[3] for f in runNNet.FLAGS) for n in ("zoneoutCell", "zoneoutHidden"))
    cfg = runNNet.run_config(runNNet._parse(["--cell", "lstm", "--zoneoutCell", "0.15", "--zoneoutHidden", "0.05"]))
    assert cfg["zoneoutCell"] == 0.15 and cfg["zoneoutHidden"] == 0.05
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f]))
    assert back["zoneoutCell"] == 0.15 and back["zoneoutHidden"] == 0.05
    assert runNNet.trained_config(f).zoneoutCell == 0.15
    old = {k: v for k, v in cfg.items() if k not in ("zoneoutCell", "zoneoutHidden")}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))
    assert back["zoneoutCell"] == 0.0 and back["zoneoutHidden"] == 0.0
    t = runNNet.trained_config(f2)
    assert t.zoneoutCell == 0.0 and t.zoneoutHidden == 0.0
