"""CPU tests of self-conditioned CTC (ctcb_brnn_config.selfCondition): the float64 restatement (tests/net_oracle.Net)
against central differences of main + lambda * intermediate on every tensor, W_c and b_c included, and at W_c = b_c = 0
against the same net without the conditioning; the config and NNet refusals; the parameter layout; the exact workspace
growth; the runNNet flag and --test."""
import ctypes

import numpy as np
import pytest

import recipes
from net_oracle import Net
from test_inter_ctc_cpu import NETS, D, K, H, _data


def _net(name, lam=0.7, round_f32=False, reg=1e-3, cond=True, wc=0.4):
    c = dict(NETS[name])
    N, tl, m = c.pop("N"), c.pop("tl"), c.pop("m")
    kw = dict(temporalLayer=tl, reg=reg, round_f32=round_f32, dropoutSeed=5, interLayer=m, interWeight=lam,
              selfCondition=cond, **c)
    np.random.seed(11)
    net = Net(D, K, H, N, 40, **kw)
    net.initParams()
    rng = np.random.RandomState(6)
    for w, b in net.stack[:N + 1]:     # no hidden unit sits exactly on its ReLU kink where a column of X is all 0
        b[...] = rng.uniform(-0.1, 0.1, b.shape)
    if net.peephole:
        rng = np.random.RandomState(4)
        for k in range(net.peep_index(0, 0), net.peep_index(0, 0) + net.entries()):
            net.stack[k][0][...] = rng.uniform(-0.5, 0.5, net.stack[k][0].shape)
    if cond and wc:
        rng = np.random.RandomState(8)
        net.stack[-1][0][...] = rng.uniform(-wc, wc, (H, K))
        net.stack[-1][1][...] = rng.uniform(-0.1, 0.1, (H, 1))
    net.dropoutStep = 2
    return net


@pytest.mark.parametrize("name", list(NETS))
def test_gradient_of_the_objective_matches_central_differences(name):
    """d(main + lambda aux)/dw of the restatement against central differences of that objective, on two entries of
    every tensor, W_c and b_c (non-zero) included."""
    net = _net(name)
    data, labels = _data()
    _, grad, skip = net.costAndGrad(data, labels)
    assert not skip and not net.interSkip and net.interCost > 0
    assert np.any(grad[-1][0]) and np.any(grad[-1][1])
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
def test_conditioning_changes_the_layers_above(name):
    """With W_c != 0 the main cost moves and the intermediate one does not (it reads X_m); at W_c = b_c = 0 the
    conditioning path adds exact zeros, so the costs and every gradient are the InterCTC net's (selfCondition off, a
    stack without [W_c, b_c]) bit for bit."""
    data, labels = _data()
    on, zero, inter = _net(name), _net(name, wc=0), _net(name, cond=False)
    c1 = on.costAndGrad(data, labels)[0]
    c0, g0, _ = zero.costAndGrad(data, labels)
    ci, gi, _ = inter.costAndGrad(data, labels)
    assert c1 != ci and on.interCost == inter.interCost
    assert c0 == ci and zero.interCost == inter.interCost and len(g0) == len(gi) + 1
    for (a, b), (x, y) in zip(g0, gi):
        assert np.array_equal(a, x) and np.array_equal(b, y)


def test_given_path_matches_own_forward():
    """costAndGradGiven with the activations, X'_m and P of the restatement's own forward pass is costAndGrad."""
    net = _net("bi_relu_m_temporal")
    data, labels = _data()
    c0, g0, _ = net.costAndGrad(data, labels)
    g0 = [[w.copy(), b.copy()] for w, b in g0]
    hActs, temporal, _ = net.forward(data)
    cond = net.conditioned(hActs)
    c1, g1, _ = net.costAndGradGiven(data, labels, hActs[1:], temporal, cond=cond)
    assert c0 == c1
    for (a, b), (x, y) in zip(g0, g1):
        assert np.allclose(a, x, rtol=1e-12, atol=1e-15) and np.allclose(b, y, rtol=1e-12, atol=1e-15)


def test_oracle_refusals():
    with pytest.raises(ValueError):
        Net(D, K, H, 3, 20, temporalLayer=2, selfCondition=True)


# ------------------------------------------------------------------------------------------------------- C ABI
def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1, 0)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _al(n):
    return (n + 255) // 256 * 256


CFG_CASES = {      # (config, interLayer, frames of layer m per utterance)
    "bi_m_temporal": (dict(), 2, 60),
    "bi_m_relu": (dict(), 1, 60),
    "uni_lstm_k2": (dict(unidirectional=1, temporalLayer=1, numTemporal=2, cell=1, peephole=1), 2, 60),
    "ln_noise_masks": (dict(layerNorm=1, weightNoise=1, maskFeatDim=41), 1, 60),
    "sub_below": (dict(subsample=3, subsampleLayer=3), 1, 60),
    "sub_at_m": (dict(subsample=3, subsampleLayer=2), 2, 20),
    "sub_stacked_above_m": (dict(subsample=2, subsampleLayer=2), 1, 60),
    "dnn": (dict(temporalLayer=0), 2, 60),
    "zoneout": (dict(cell=1, zoneout=1), 1, 60),
}


@pytest.mark.parametrize("name", list(CFG_CASES))
def test_parameter_layout(name):
    from _ctcb import lib
    kw, m, _ = CFG_CASES[name]
    off = _cfg(interLayer=m, interWeight=0.3, **kw)
    on = _cfg(interLayer=m, interWeight=0.3, selfCondition=1, **kw)
    assert off.selfCondition == 0     # an initialiser without the member keeps its meaning
    n0, n1 = lib.ctcb_brnn_num_tensors(ctypes.byref(off)), lib.ctcb_brnn_num_tensors(ctypes.byref(on))
    assert n1 == n0 + 2
    o, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    for idx in range(n0):     # every other tensor where it was
        a = []
        for cfg in (off, on):
            assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), idx, ctypes.byref(o), ctypes.byref(r),
                                             ctypes.byref(c)) == 0
            a.append((o.value, r.value, c.value))
        assert a[0] == a[1], idx
    P0 = lib.ctcb_brnn_param_count(ctypes.byref(off))
    Hc, Kc = on.layerSize, on.outputDim
    lib.ctcb_brnn_tensor_info(ctypes.byref(on), n0, ctypes.byref(o), ctypes.byref(r), ctypes.byref(c))
    assert (o.value, r.value, c.value) == ((P0 + 3) // 4 * 4, Hc, Kc)
    wc = o.value
    lib.ctcb_brnn_tensor_info(ctypes.byref(on), n0 + 1, ctypes.byref(o), ctypes.byref(r), ctypes.byref(c))
    assert (o.value, r.value, c.value) == ((wc + Hc * Kc + 3) // 4 * 4, Hc, 1)
    assert lib.ctcb_brnn_param_count(ctypes.byref(on)) == o.value + Hc
    assert lib.ctcb_brnn_tensor_info(ctypes.byref(on), n0 + 2, ctypes.byref(o), None, None) == -1


@pytest.mark.parametrize("name", list(CFG_CASES))
def test_workspace_grows_by_exactly_the_conditioning_buffers(name):
    from _ctcb import lib
    kw, m, Tm = CFG_CASES[name]
    off = _cfg(interLayer=m, interWeight=0.3, **kw)
    on = _cfg(interLayer=m, interWeight=0.3, selfCondition=1, **kw)
    base = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    assert base > 0
    B, Kc, Hc = on.maxB, on.outputDim, on.layerSize
    RmK = _al(Tm * B * Kc * 4)
    # the noisy copy of weightNoise = 1 holds W_c and b_c too; everything behind it moves by as much
    moved = 0
    if on.weightNoise:
        moved = _al(4 * lib.ctcb_brnn_param_count(ctypes.byref(on))) - _al(4 * lib.ctcb_brnn_param_count(ctypes.byref(off)))
        assert moved > 0
    base += moved
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) == base + _al(Tm * B * Hc * 4) + 2 * RmK
    fb = lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), None)
    assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(on), None) == fb + 2 * RmK
    assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(on)) == lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))
    for what in range(12):
        for layer in range(5):
            a, b = ctypes.c_size_t(), ctypes.c_size_t()
            ra = lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, layer, ctypes.byref(a), None)
            rb = lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, layer, ctypes.byref(b), None)
            assert ra == rb and a.value + (moved if what >= 8 else 0) == b.value, (what, layer)
    offs, widths = [], []
    for what in range(12, 15):
        o, w = ctypes.c_size_t(), ctypes.c_int32()
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, 0, ctypes.byref(o), ctypes.byref(w)) == 0
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, 0, ctypes.byref(o), None) == -1
        offs.append(o.value)
        widths.append(w.value)
    assert offs == [base, base + _al(Tm * B * Hc * 4), base + _al(Tm * B * Hc * 4) + RmK]
    assert widths == [Hc, Kc, Kc]


def test_config_refusals():
    from _ctcb import lib
    for kw, text in ((dict(selfCondition=1), b"needs interLayer"),
                     (dict(selfCondition=2, interLayer=1, interWeight=0.5), b"selfCondition 2"),
                     (dict(selfCondition=-1, interLayer=1, interWeight=0.5), b"selfCondition -1")):
        cfg = _cfg(**kw)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, kw
        assert lib.ctcb_brnn_num_tensors(ctypes.byref(cfg)) == 0, kw
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, kw
        assert text in lib.ctcb_last_error(), (kw, lib.ctcb_last_error())


def test_softmax_backward_argument_checks():
    from _ctcb import lib
    buf = ctypes.create_string_buffer(64)
    for args, text in (((None, buf, None, buf, 1, 1), b"null pointer"), ((buf, None, None, buf, 1, 1), b"null pointer"),
                       ((buf, buf, None, None, 1, 1), b"null pointer"), ((buf, buf, None, buf, 0, 1), b"R = 0"),
                       ((buf, buf, None, buf, 1, 0), b"K = 0"), ((buf, buf, None, buf, 1 << 40, 4), b"need 1 <= R")):
        assert lib.ctcb_softmax_rows_backward_f32(*args, None) == -1, args
        assert text in lib.ctcb_last_error(), (args, lib.ctcb_last_error())


def test_nnet_refusals():
    import nnets.brnnet as brnnet
    import nnets.nnet as nnet
    import nnets.rnnet as rnnet
    for cls in (brnnet.NNet, rnnet.NNet, nnet.NNet):
        with pytest.raises(ValueError, match="needs interLayer"):
            cls(13, 11, 16, 3, 20, selfCondition=True)


def test_checkpoint_pair_check():
    """fromFile's count check, on the host: a self-conditioned net refuses a checkpoint without [W_c, b_c], and a net
    without it refuses one with it, naming both tensor counts."""
    import nnets.brnnet as brnnet
    net = brnnet.NNet.__new__(brnnet.NNet)
    net.layerSize, net.outputDim, net.cell, net.numTemporal, net.layerNorm = H, K, "relu", 1, False
    views = [[np.zeros((H, D)), np.zeros((H, 1))], [np.zeros((K, H)), np.zeros((K, 1))]]
    cond = [[np.zeros((H, K)), np.zeros((H, 1))]]
    net.selfCondition = True
    with pytest.raises(ValueError, match="has 4 tensors where this net \\(selfCondition=True\\) has 6"):
        net.check_pair_count(views, views + cond, "stack")
    net.check_pair_count(views + cond, views + cond, "stack")
    net.selfCondition = False
    with pytest.raises(ValueError, match="has 6 tensors where this net \\(selfCondition=False\\) has 4"):
        net.check_pair_count(views + cond, views, "stack")
    net.check_pair_count(views, views, "stack")


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).selfCondition is False
    assert any(f[0] == "selfCondition" and f[3] for f in runNNet.FLAGS) and "--selfCondition" in runNNet.__doc__
    cfg = runNNet.run_config(runNNet._parse(["--interLayer", "2", "--interWeight", "0.43", "--selfCondition"]))
    assert cfg["selfCondition"] is True
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["selfCondition"] is True
    old = {k: v for k, v in cfg.items() if k != "selfCondition"}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["selfCondition"] is False
    assert runNNet.trained_config(f2).selfCondition is False


@pytest.mark.parametrize("cond", [False, True])
def test_test_mode_builds_the_conditioned_net(tmp_path, monkeypatch, cond):
    """--test passes interLayer, interWeight and selfCondition to the net only when the trained config conditions."""
    import runNNet
    from run_utils import dump_config
    cfg = runNNet.run_config(runNNet._parse(["--interLayer", "2", "--interWeight", "0.43"]
                                            + (["--selfCondition"] if cond else [])))
    cfg["in_file"] = str(tmp_path / "params.bin")
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    seen = {}

    class Stop(Exception):
        pass

    def fake(*args, **kw):
        seen.update(kw)
        raise Stop

    monkeypatch.setattr(runNNet.rnnet, "NNet", fake)
    with pytest.raises(Stop):
        runNNet.test(runNNet._parse(["--cfg_file", f, "--test"]))
    if cond:
        assert seen["selfCondition"] is True and seen["interLayer"] == 2 and seen["interWeight"] == 0.43
    else:
        assert "selfCondition" not in seen and "interLayer" not in seen
    assert seen["train"] is False
