"""CPU tests of layer normalisation (ctcb_brnn_config.layerNorm = 1): the config contract of the library (tensor table,
both workspaces, refusal of bad values) and runNNet's --layerNorm flag (the float64 restatement of the net is tested
in tests/test_net_oracle_cpu.py)."""
import ctypes

import pytest

from test_lstm_cpu import _training_ws


def _cfg(D, K, H, N, tl, T, B, L, uni=0, nt=1, cell=0, ln=1):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, T, B, L, 0.0, 20.0, uni, nt, cell, ln)


def _layout(cfg):
    from _ctcb import lib
    n = lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for i in range(n):
        assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        out.append((off.value, r.value, c.value))
    return out


def _fwd_ws(cfg):
    from _ctcb import lib
    f = ctypes.c_size_t()
    return lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), ctypes.byref(f)), f.value


def _normed(N, tl, nt):
    return [i for i in range(1, N + 1) if not (tl > 0 and tl <= i < tl + nt)]


# (D, K, H, N, tl, T, B, L, uni, nt, cell): C2, a stack, a DNN, an LSTM net, a uni-directional net with odd H
NETS = [(41, 62, 512, 2, 1, 200, 32, 30, 0, 1, 0), (13, 11, 70, 4, 2, 37, 5, 9, 0, 2, 0),
        (13, 11, 64, 3, 0, 40, 4, 9, 0, 1, 0), (13, 11, 64, 3, 2, 60, 8, 20, 1, 1, 1),
        (41, 32, 1824, 5, 3, 50, 4, 20, 1, 1, 0)]


# ------------------------------------------------------------------------------------------- the config contract
@pytest.mark.parametrize("net", NETS)
def test_layer_norm_off_is_the_config_without_the_member(net):
    """layerNorm = 0 and a config that never sets it (ctypes zero-fills it) report the same everything, and the same as
    the restatement of the workspace of a net without normalisation."""
    import _ctcb
    from _ctcb import lib
    args = net[:8] + (0.0, 20.0, net[8], net[9], net[10])
    a, b = _ctcb.BrnnConfig(*args), _ctcb.BrnnConfig(*args)
    b.layerNorm = 0
    assert a.layerNorm == 0
    assert _layout(a) == _layout(b)
    for q in (lib.ctcb_brnn_param_count, lib.ctcb_brnn_num_tensors, lib.ctcb_brnn_workspace_bytes,
              lib.ctcb_brnn_error_flag_offset):
        assert q(ctypes.byref(a)) == q(ctypes.byref(b))
    assert _fwd_ws(a) == _fwd_ws(b)
    if net[4] > 0:      # the restatement covers nets with a temporal layer
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(a)) == _training_ws(*net)


def test_invalid_layer_norm_is_refused_with_a_message():
    from _ctcb import lib
    for bad in (2, -1, 7):
        cfg = _cfg(13, 11, 64, 3, 2, 60, 8, 20, ln=bad)
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
        assert ("layerNorm %d" % bad) in lib.ctcb_last_error().decode()
        assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0
    cfg = _cfg(13, 11, 8193, 2, 1, 4, 2, 2)           # wider than the kernels hold a row
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert "layerSize <= 8192" in lib.ctcb_last_error().decode()
    cfg.layerNorm = 0
    assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) > 0


@pytest.mark.parametrize("net", NETS)
def test_pairs_go_behind_every_old_tensor(net):
    from _ctcb import lib
    D, K, H, N, tl, T, B, L, uni, nt, cell = net
    off, on = _layout(_cfg(*net, ln=0)), _layout(_cfg(*net, ln=1))
    normed = _normed(N, tl, nt)
    assert on[:len(off)] == off                       # every old tensor keeps its offset and shape
    assert len(on) == len(off) + 2 * len(normed)
    assert [(r, c) for _, r, c in on[len(off):]] == [(H, 1)] * (2 * len(normed))
    for (o0, r0, c0), (o1, _, _) in zip(on, on[1:]):
        assert o1 == (o0 + r0 * c0 + 3) // 4 * 4
    assert lib.ctcb_brnn_param_count(ctypes.byref(_cfg(*net))) == (on[-1][0] + H + 3) // 4 * 4


@pytest.mark.parametrize("net", NETS)
def test_training_workspace_follows_the_formula(net):
    """z, mu and rstd of every normalised layer and the partial area, behind the layout without normalisation; the
    forward workspace does not grow."""
    from _ctcb import lib
    D, K, H, N, tl, T, B, L, uni, nt, cell = net
    al = lambda x: (x + 255) // 256 * 256     # noqa: E731
    R = T * B
    parts = min(1024, -(-R // 8))
    grow = len(_normed(N, tl, nt)) * (al(R * H * 4) + 2 * al(R * 4)) + al(2 * parts * H * 4)
    off, on = _cfg(*net, ln=0), _cfg(*net, ln=1)
    assert lib.ctcb_layernorm_workspace_bytes(R, H) == al(2 * parts * H * 4)
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) == lib.ctcb_brnn_workspace_bytes(ctypes.byref(off)) + grow
    assert _fwd_ws(on) == _fwd_ws(off)
    assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(on)) == lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))


def test_growth_at_c2_and_c3():
    """The training workspace grows by z, mu, rstd of the normalised layers and the partials: 13.2 MB + 3.3 MB at C2
    (one normalised layer of 6400 x 512, 800 row chunks) and 0.78 GiB + 8 MiB at C3 (two of 102400 x 1024)."""
    from _ctcb import lib
    grow = {}
    for name, net in (("c2", (41, 62, 512, 2, 1, 200, 32, 30, 0, 1, 0)), ("c3", (41, 32, 1024, 3, 2, 800, 128, 100, 0, 1, 0))):
        grow[name] = lib.ctcb_brnn_workspace_bytes(ctypes.byref(_cfg(*net))) - \
            lib.ctcb_brnn_workspace_bytes(ctypes.byref(_cfg(*net, ln=0)))
    assert grow["c2"] == 6400 * 512 * 4 + 2 * 6400 * 4 + 2 * 800 * 512 * 4, grow
    assert grow["c3"] == 2 * (102400 * 1024 * 4 + 2 * 102400 * 4) + 2 * 1024 * 1024 * 4, grow
    assert 0.78 < grow["c3"] / 2 ** 30 < 0.80, grow


def test_entry_points_check_their_arguments():
    from _ctcb import lib
    assert lib.ctcb_layernorm_workspace_bytes(100, 0) == 0
    assert lib.ctcb_layernorm_workspace_bytes(100, 8193) == 0
    assert lib.ctcb_layernorm_forward_f32(None, None, None, None, None, None, 4, 64, None) == -1
    assert "null pointer" in lib.ctcb_last_error().decode()
    assert lib.ctcb_layernorm_forward_f32(None, None, None, None, None, None, 4, 9000, None) == -1
    assert "H = 9000" in lib.ctcb_last_error().decode()
    assert lib.ctcb_layernorm_backward_f32(None, None, None, None, None, None, None, 4, 64, 0, None, 0, None) == -1


# ------------------------------------------------------------------------------------------- runNNet
def test_runnnet_layer_norm_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).layerNorm is False
    assert runNNet._parse(["--layerNorm"]).layerNorm is True
    cfg = runNNet.run_config(runNNet._parse(["--layerNorm"]))
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.trained_config(f).layerNorm is True                                  # --test rebuilds it
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["layerNorm"] is True    # resume keeps it
    old = dict(cfg)
    del old["layerNorm"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.trained_config(f2).layerNorm is False                 # a model from before the flag
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["layerNorm"] is False
