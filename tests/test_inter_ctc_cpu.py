"""CPU tests of the intermediate CTC loss (ctcb_brnn_config.interLayer): the float64 restatement
(tests/net_oracle.Net) against central differences of its objective, its intermediate term against the head net's loss,
each CTC skipping on its own; the config and NNet refusals; the exact workspace growth; the runNNet flags."""
import ctypes

import numpy as np
import pytest

import recipes
from net_oracle import Net

D, K, H = 5, 6, 6
NETS = {
    "bi_relu_m_temporal": dict(N=3, tl=2, m=2),
    "uni_relu_m_relu": dict(N=3, tl=2, m=1, unidirectional=True),
    "lstm_peep_k2_m_temporal": dict(N=4, tl=2, m=3, numTemporal=2, cell="lstm", peephole=True),
    "uni_lstm_m_below": dict(N=3, tl=2, m=1, unidirectional=True, cell="lstm"),
    "ln_drop_m_relu": dict(N=3, tl=3, m=2, layerNorm=True, dropout=0.3, allowTopTemporal=True),
    "sub_below": dict(N=3, tl=2, m=1, subsample=2, subsampleLayer=3),
    "sub_stacked_above_m": dict(N=3, tl=2, m=1, subsample=2, subsampleLayer=2),
    "sub_above": dict(N=3, tl=1, m=2, subsample=3, subsampleLayer=2),
    "dnn": dict(N=3, tl=-1, m=2),
}


def _net(name, lam=0.7, round_f32=False, reg=1e-3):
    c = dict(NETS[name])
    N, tl, m = c.pop("N"), c.pop("tl"), c.pop("m")
    kw = dict(temporalLayer=tl, reg=reg, round_f32=round_f32, dropoutSeed=5, interLayer=m if lam else 0,
              interWeight=lam, **c)
    np.random.seed(11)
    net = Net(D, K, H, N, 40, **kw)
    net.initParams()
    rng = np.random.RandomState(6)
    for w, b in net.stack[:N + 1]:     # no hidden unit sits exactly on its ReLU kink where a column of X is all 0
        b[...] = rng.uniform(-0.1, 0.1, b.shape)
    if net.peephole:
        rng = np.random.RandomState(4)
        for k in range(len(net.stack) - net.entries(), len(net.stack)):
            net.stack[k][0][...] = rng.uniform(-0.5, 0.5, net.stack[k][0].shape)
    net.dropoutStep = 2
    return net


def _data(T=12, L=3, seed=3):
    datas, labelss = recipes.synth_batch(D, K, [T], [L], seed=seed)
    return datas[0], labelss[0]


@pytest.mark.parametrize("name", list(NETS))
def test_gradient_of_the_objective_matches_central_differences(name):
    """d(main + lambda aux)/dw of the float64 restatement against central differences of that objective, on two
    entries of every tensor (the intermediate term is not zero: the head's gradient reaches every tensor below m)."""
    net = _net(name)
    data, labels = _data()
    _, grad, skip = net.costAndGrad(data, labels)
    assert not skip and not net.interSkip and net.interCost > 0
    eps = 1e-6
    for k, (w, b) in enumerate(net.stack):
        for arr, g in ((w, grad[k][0]), (b, grad[k][1])):
            if arr.shape == (1, 1):
                continue
            for idx in (tuple(s // 2 for s in arr.shape), tuple(s - 1 for s in arr.shape)):
                old = arr[idx]
                arr[idx] = old + eps
                up = net.objective(data, labels)
                arr[idx] = old - eps
                dn = net.objective(data, labels)
                arr[idx] = old
                assert abs((up - dn) / (2 * eps) - g[idx]) <= 1e-5 * max(1.0, abs(g[idx])), (k, idx)


@pytest.mark.parametrize("name", list(NETS))
def test_intermediate_term_is_the_head_nets_loss_and_reaches_only_the_head(name):
    """The objective minus the main cost is lambda times the head's CTC loss; tensors above layer m other than the
    output map get exactly the main gradient."""
    with_ = _net(name)
    without = _net(name, lam=0.0)
    data, labels = _data()
    c1, g1, _ = with_.costAndGrad(data, labels)
    c0, g0, _ = without.costAndGrad(data, labels)
    assert c1 == c0
    net, index = with_.head()
    A = with_.stack[with_.numLayers][0].dot(with_.forward(data)[0][with_.interLayer]) + with_.stack[with_.numLayers][1]
    assert np.isclose(with_.interCost, net.costAndGrad(data, labels)[0], rtol=1e-12)
    assert A.shape == (K, net.forward(data)[0][-1].shape[1])
    for t in range(len(g0)):
        if t not in index:
            assert np.array_equal(g1[t][0], g0[t][0]) and np.array_equal(g1[t][1], g0[t][1]), t
    assert not np.array_equal(g1[with_.numLayers][0], g0[with_.numLayers][0])


def test_each_ctc_skips_on_its_own():
    """Below the subsampling point the intermediate CTC has T frames where the main one has ceil(T / 2): five equal
    labels need nine frames, so the main CTC alone skips that utterance, which still gets the intermediate gradient."""
    net = _net("sub_below")
    datas, _ = recipes.synth_batch(D, K, [12, 12], [1, 1], seed=3)
    labelss = [np.array([1, 2, 3], np.int32), np.array([3] * 5, np.int32)]
    costs, grad, skips = net.costAndGradBatch(datas, labelss)
    assert list(skips) == [False, True] and list(net.interSkips) == [False, False]
    _, g, s = net.costAndGrad(datas[1], labelss[1])
    assert s and any(np.any(gw) for gw, _ in g)


def test_oracle_refusals():
    for kw in (dict(interLayer=1), dict(interLayer=1, interWeight=float("nan")), dict(interWeight=0.5),
               dict(interLayer=3, interWeight=0.5), dict(interLayer=-1, interWeight=0.5),
               dict(interLayer=1, interWeight=0.5, subsample=2, subsampleLayer=4)):
        with pytest.raises(ValueError):
            Net(D, K, H, 3, 20, temporalLayer=2, **kw)


# ------------------------------------------------------------------------------------------------------- C ABI
def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _al(n):
    return (n + 255) // 256 * 256


CFG_CASES = {      # (config, interLayer, rows of layer m per utterance, whether the CTC area is its own)
    "bi_m_temporal": (dict(), 2, 60, False),
    "bi_m_relu": (dict(), 1, 60, False),
    "uni_lstm_k2": (dict(unidirectional=1, temporalLayer=1, numTemporal=2, cell=1, peephole=1), 2, 60, False),
    "ln_noise_masks": (dict(layerNorm=1, weightNoise=1, maskFeatDim=41), 1, 60, False),
    "sub_below": (dict(subsample=3, subsampleLayer=3), 1, 60, True),
    "sub_at_m": (dict(subsample=3, subsampleLayer=2), 2, 20, False),
    "sub_stacked_above_m": (dict(subsample=2, subsampleLayer=2), 1, 60, True),
    "dnn": (dict(temporalLayer=0), 2, 60, False),
    "zoneout": (dict(cell=1, zoneout=1), 1, 60, False),
}


@pytest.mark.parametrize("name", list(CFG_CASES))
def test_workspace_grows_by_exactly_the_intermediate_buffers(name):
    from _ctcb import lib
    kw, m, Tm, own_ctc = CFG_CASES[name]
    off = _cfg(**kw)
    assert off.interLayer == 0        # an initialiser without the members keeps its meaning
    on = _cfg(interLayer=m, interWeight=0.3, **kw)
    base = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    assert base > 0
    B, Kc = on.maxB, on.outputDim
    grow = 2 * _al(Tm * B * Kc * 4) + 2 * _al(B * 4)
    if own_ctc:
        grow += _al(lib.ctcb_ctc_workspace_bytes(B, on.maxT, on.maxLabels))
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) == base + grow
    assert lib.ctcb_brnn_param_count(ctypes.byref(on)) == lib.ctcb_brnn_param_count(ctypes.byref(off))
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(on)) == lib.ctcb_brnn_num_tensors(ctypes.byref(off))
    assert (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(on), None)
            == lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), None))
    assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(on)) == lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))
    for what in range(8):
        for layer in range(5):
            a, b = ctypes.c_size_t(), ctypes.c_size_t()
            ra = lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, layer, ctypes.byref(a), None)
            rb = lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, layer, ctypes.byref(b), None)
            assert ra == rb and a.value == b.value, (what, layer)
    # the new entries lie behind everything the net without the loss has, in the order the header gives
    offs, widths = [], []
    for what in range(8, 12):
        o, w = ctypes.c_size_t(), ctypes.c_int32()
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, 0, ctypes.byref(o), ctypes.byref(w)) == 0
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, 0, ctypes.byref(o), None) == -1
        offs.append(o.value)
        widths.append(w.value)
    assert offs[0] == base and widths == [Kc, Kc, 1, 1]
    assert offs[1] == base + _al(Tm * B * Kc * 4) and offs[3] == offs[2] + _al(B * 4)


def test_config_refusals():
    from _ctcb import lib
    for kw, text in ((dict(interLayer=3, interWeight=0.5), b"interLayer 3"),
                     (dict(interLayer=-1, interWeight=0.5), b"interLayer -1"),
                     (dict(interLayer=1, interWeight=0.0), b"interWeight 0"),
                     (dict(interLayer=1, interWeight=-1.0), b"interWeight -1"),
                     (dict(interLayer=1, interWeight=float("nan")), b"not a finite"),
                     (dict(interLayer=1, interWeight=float("inf")), b"not a finite"),
                     (dict(interLayer=1, interWeight=0.5, subsample=2, subsampleLayer=4), b"stacked frames"),
                     (dict(interLayer=1, interWeight=0.5, numLayers=1, temporalLayer=1), b"interLayer 1")):
        cfg = _cfg(**kw)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, kw
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, kw
        assert text in lib.ctcb_last_error(), (kw, lib.ctcb_last_error())
    # the weight is ignored without the layer, as subsampleLayer is without subsampling
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(_cfg(interWeight=float("nan")))) == \
        lib.ctcb_brnn_workspace_bytes(ctypes.byref(_cfg()))


def test_nnet_refusals():
    import nnets.brnnet as brnnet
    import nnets.nnet as nnet
    import nnets.rnnet as rnnet
    for cls in (brnnet.NNet, rnnet.NNet):
        with pytest.raises(ValueError, match="interWeight > 0"):
            cls(13, 11, 16, 3, 20, temporalLayer=2, interLayer=1)
        with pytest.raises(ValueError, match="interWeight > 0"):
            cls(13, 11, 16, 3, 20, temporalLayer=2, interLayer=1, interWeight=float("inf"))
        with pytest.raises(ValueError, match="needs interLayer"):
            cls(13, 11, 16, 3, 20, temporalLayer=2, interWeight=0.3)
    with pytest.raises(ValueError, match="interWeight > 0"):
        nnet.NNet(13, 11, 16, 3, 20, interLayer=2, interWeight=-0.5)


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    opts = runNNet._parse([])
    assert opts.interLayer == 0 and opts.interWeight == 0.0
    assert all(any(f[0] == n and f[3] for f in runNNet.FLAGS) for n in ("interLayer", "interWeight"))
    assert "--interLayer" in runNNet.__doc__ and "--interWeight" in runNNet.__doc__
    cfg = runNNet.run_config(runNNet._parse(["--interLayer", "2", "--interWeight", "0.43"]))
    assert cfg["interLayer"] == 2 and cfg["interWeight"] == 0.43
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f]))
    assert back["interLayer"] == 2 and back["interWeight"] == 0.43
    old = {k: v for k, v in cfg.items() if k not in ("interLayer", "interWeight")}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))
    assert back["interLayer"] == 0 and back["interWeight"] == 0.0
    t = runNNet.trained_config(f2)
    assert t.interLayer == 0 and t.interWeight == 0.0
