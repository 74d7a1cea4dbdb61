"""CPU tests of stacked temporal layers (ctcb_brnn_config.numTemporal): the flat layout and both workspace sizes the
library reports, the rejection of blocks that do not fit, and the runNNet flag (the float64 restatement of the
stacked net is tested in tests/test_net_oracle_cpu.py).  No compute call is made on a device here."""
import ctypes

import pytest

# (D, K, H, N, tl, T, B, L, uni)
NETS = [(41, 62, 512, 2, 1, 200, 32, 30, 0), (13, 11, 64, 3, 2, 60, 8, 20, 1), (41, 32, 1024, 3, 2, 800, 8, 100, 0),
        (13, 11, 96, 4, 1, 37, 5, 9, 0), (13, 11, 64, 2, 0, 60, 8, 20, 0), (13, 11, 64, 2, 3, 60, 8, 20, 0),
        (41, 62, 512, 1, 1, 200, 32, 30, 0)]


def _cfg(D, K, H, N, tl, T, B, L, uni, *nt):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, T, B, L, 0.0, 20.0, uni, *nt)


def _layout(cfg):
    from _ctcb import lib
    nt = lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for i in range(nt):
        assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        out.append((off.value, r.value, c.value))
    return out


def _sizes(cfg):
    from _ctcb import lib
    flag = ctypes.c_size_t()
    return (lib.ctcb_brnn_num_tensors(ctypes.byref(cfg)), lib.ctcb_brnn_param_count(ctypes.byref(cfg)),
            lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)), lib.ctcb_brnn_error_flag_offset(ctypes.byref(cfg)),
            lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), ctypes.byref(flag)), flag.value)


def _act(cfg, what, layer):
    from _ctcb import lib
    off, w = ctypes.c_size_t(), ctypes.c_int32()
    rc = lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), what, layer, ctypes.byref(off), ctypes.byref(w))
    return rc, off.value, w.value


@pytest.mark.parametrize("net", NETS)
def test_zero_and_one_temporal_layer_are_todays_net(net):
    base = _cfg(*net)
    for k in (0, 1):
        cfg = _cfg(*net, k)
        assert _sizes(cfg) == _sizes(base)
        assert _layout(cfg) == _layout(base)
        for what in (0, 1, 2):
            for layer in range(0, net[3] + 3):
                assert _act(cfg, what, layer) == _act(base, what, layer)


@pytest.mark.parametrize("uni", [0, 1])
@pytest.mark.parametrize("k", [2, 3])
def test_stacked_layout_order_and_alignment(k, uni):
    D, K, H, N, tl = 13, 11, 30, 4, 1        # H*H = 900 floats: every tensor is followed by an alignment gap
    cfg = _cfg(D, K, H, N, tl, 40, 4, 9, uni, k)
    lay = _layout(cfg)
    nrec = 1 if uni else 2
    assert len(lay) == 2 * (N + 1) + 2 * nrec * k
    assert lay[:2 * (N + 1)] == _layout(_cfg(D, K, H, N, tl, 40, 4, 9, uni))[:2 * (N + 1)]
    shapes = [(r, c) for _, r, c in lay]
    assert shapes[2 * (N + 1):] == [(H, H), (1, 1)] * (nrec * k)
    offs = [o for o, _, _ in lay]
    assert all(o % 4 == 0 for o in offs)
    for (o, r, c), (o2, _, _) in zip(lay, lay[1:]):     # ascending, packed up to the 16-byte alignment
        assert o2 == (o + r * c + 3) // 4 * 4
    o, r, c = lay[-1]
    from _ctcb import lib
    assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == (o + r * c + 3) // 4 * 4


@pytest.mark.parametrize("uni", [0, 1])
@pytest.mark.parametrize("net", [(13, 11, 64, 4, 1, 60, 8, 20), (41, 32, 1024, 4, 2, 37, 3, 10),
                                 (13, 11, 96, 3, 1, 33, 5, 9)])
def test_training_workspace_grows_by_the_documented_formula(net, uni):
    """k > 1: every temporal layer above the first adds For_j (and Back_j), and the stack adds a second dFor / dBack
    pair -- k * (2 bi-directional, 1 uni-directional) buffers of maxT*maxB*H floats, each rounded up to 256 bytes.
    The forward-only workspace does not grow."""
    D, K, H, N, tl, T, B, L = net
    one = _sizes(_cfg(*net, uni, 1))
    per_buf = (T * B * H * 4 + 255) // 256 * 256
    for k in range(2, N - tl + 2):
        got = _sizes(_cfg(*net, uni, k))
        assert got[2] - one[2] == k * (1 if uni else 2) * per_buf, k
        assert got[4] == one[4] and got[5] == one[5]            # forward-only layout and its error flag
        assert got[3] > one[3]                                  # the training error flag sits behind the new buffers


def test_activation_offsets_of_stacked_layers():
    net = (13, 11, 64, 4, 1, 60, 8, 20)
    for uni in (0, 1):
        cfg = _cfg(*net, uni, 3)
        ws = _sizes(cfg)[2]
        fors = [_act(cfg, 1, layer) for layer in (1, 2, 3)]
        assert all(rc == 0 and w == 64 for rc, _, w in fors)
        offs = [o for _, o, _ in fors]
        if not uni:
            backs = [_act(cfg, 2, layer) for layer in (1, 2, 3)]
            assert all(rc == 0 and w == 64 for rc, _, w in backs)
            offs += [o for _, o, _ in backs]
        else:
            assert _act(cfg, 2, 2)[0] == -1
        offs += [_act(cfg, 0, i)[1] for i in range(1, 6)]
        assert len(set(offs)) == len(offs) and all(o + 60 * 8 * 64 * 4 <= ws for o in offs)
        assert _act(cfg, 1, 4)[0] == -1 and _act(cfg, 1, 0)[0] == -1     # outside the block


@pytest.mark.parametrize("tl,k,N", [(0, 2, 3), (-1, 2, 3), (2, 3, 3), (3, 2, 3), (1, 5, 4), (5, 2, 4)])
def test_blocks_that_do_not_fit_are_rejected(tl, k, N):
    import _ctcb
    from _ctcb import lib
    cfg = _cfg(13, 11, 64, N, tl, 60, 8, 20, 0, k)
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(cfg)) == 0
    assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == 0
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0
    assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == 0
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert b"temporal layers" in lib.ctcb_last_error()
    with pytest.raises(ValueError):
        _ctcb.check(-1)
    # a negative count is no count at all
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(_cfg(13, 11, 64, 3, 1, 60, 8, 20, 0, -1))) == 0
    # the block may end at the top hidden layer
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(_cfg(13, 11, 64, 3, 2, 60, 8, 20, 0, 2))) == 2 * 4 + 8


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_num_temporal_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    cli = runNNet._parse([])
    assert cli.numTemporal == 1
    cfg = runNNet.run_config(runNNet._parse(["--numTemporal", "2", "--numLayers", "4", "--temporalLayer", "1"]))
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.trained_config(f).numTemporal == 2
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["numTemporal"] == 2       # resume keeps it
    old = dict(cfg)
    del old["numTemporal"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.trained_config(f2).numTemporal == 1                  # --test of a model from before the flag
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["numTemporal"] == 1      # and its resume
