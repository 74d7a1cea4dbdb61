"""CPU tests of the LSTM cell (ctcb_brnn_config.cell = 1): the config contract the library reports -- an invalid
cell, the tensor layout, the training workspace against its formula, the runNNet flag and an old cfg.json (the float64
restatement of the net is tested in tests/test_net_oracle_cpu.py).  No compute call is made on a device here."""
import ctypes

import pytest


def _cfg(D, K, H, N, tl, T, B, L, uni=0, nt=1, cell=1):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, T, B, L, 0.0, 20.0, uni, nt, cell)


def _layout(cfg):
    from _ctcb import lib
    n = lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    out = []
    for i in range(n):
        assert lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        out.append((off.value, r.value, c.value))
    return out


# ------------------------------------------------------------------------------------------- the config contract
def test_invalid_cell_is_refused_with_a_message():
    import _ctcb
    lib = _ctcb.lib
    for bad in (2, -1, 7):
        cfg = _cfg(13, 11, 64, 3, 2, 60, 8, 20, cell=bad)
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
        assert ("cell %d" % bad) in lib.ctcb_last_error().decode()
        assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0


@pytest.mark.parametrize("uni", [0, 1])
@pytest.mark.parametrize("nt", [1, 2, 3])
def test_lstm_tensor_layout(uni, nt):
    """The tensors are packed at 16-byte alignment, and only the temporal maps and the recurrent matrices differ from
    the relu config's (test_net_oracle_cpu.py checks every shape against the float64 restatement)."""
    D, K, H, N, tl = 13, 11, 70, 4, 2
    cfg = _cfg(D, K, H, N, tl, 60, 8, 20, uni, nt)
    lay = _layout(cfg)
    for (o0, r0, c0), (o1, _, _) in zip(lay, lay[1:]):
        assert o1 == (o0 + r0 * c0 + 3) // 4 * 4
    from _ctcb import lib
    assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == (lay[-1][0] + 1 + 3) // 4 * 4
    # the relu config of the same sizes: the same number of tensors, only the shapes of the temporal ones change
    relu = _layout(_cfg(D, K, H, N, tl, 60, 8, 20, uni, nt, cell=0))
    assert len(relu) == len(lay)
    for i, ((_, r, c), (_, r0, c0)) in enumerate(zip(lay, relu)):
        temporal_map = i < 2 * (N + 1) and tl <= i // 2 + 1 < tl + nt
        if temporal_map:
            assert (r, c) == ((1 if uni else 2) * 4 * H, c0)
        elif i >= 2 * (N + 1) and i % 2 == 0:
            assert (r, c) == (4 * H, H)
        else:
            assert (r, c) == (r0, c0)


def _training_ws(D, K, H, N, tl, T, B, L, uni, nt, cell):
    """ws_layout of brnn.cu restated: every area rounded up to 256 bytes, in the order the library lays them out."""
    from _ctcb import lib
    al = lambda x: (x + 255) // 256 * 256
    R = T * B
    G = (1 if uni else 2) * 4 * H
    temporal = lambda i: tl > 0 and tl <= i < tl + nt
    size = lambda i: D if i == 0 else (H if i <= N else K)
    rows = lambda i: G if cell and temporal(i) else size(i)
    RH = R * H * 4
    tot = sum(al(R * rows(i) * 4) for i in range(1, N + 2))
    tot += 4 * al(RH) + (nt - 1) * (1 if uni else 2) * al(RH) + ((1 if uni else 2) * al(RH) if nt > 1 else 0)
    if cell:
        tot += nt * (1 if uni else 3) * al(RH)          # c per direction, and For + Back when bi-directional
    wide = max(H, K)
    wide_g = max(wide, G) if cell else wide
    tot += sum(al(R * (wide_g if rows(j) != size(j) else wide) * 4) for j in range(1, N + 2))
    tot += al(lib.ctcb_ctc_workspace_bytes(B, T, L))
    g = 0
    for i in range(N + 1):
        g = max(g, lib.ctcb_gemm_workspace_bytes(R, rows(i + 1), size(i)), lib.ctcb_gemm_workspace_bytes(R, size(i), rows(i + 1)),
                lib.ctcb_gemm_workspace_bytes(rows(i + 1), size(i), R))
    g = max(g, lib.ctcb_gemm_pair_workspace_bytes(4 * H if cell else H, H, R))
    tot += 2 * al(g)
    tot += 2 * al(-(-R // 128) * wide_g * 4) + al(8192) + al(4096)
    tot += al(2 * B * H * 4) if cell else al(lib.ctcb_brnn_sweep_workspace_bytes(H, B) - 4096)
    return tot


@pytest.mark.parametrize("net", [(41, 62, 512, 2, 1, 200, 32, 30, 0, 1), (13, 11, 64, 3, 2, 60, 8, 20, 1, 1),
                                 (13, 11, 70, 4, 2, 37, 5, 9, 0, 3), (41, 32, 1024, 3, 2, 80, 8, 30, 0, 2),
                                 (13, 300, 64, 3, 1, 40, 4, 9, 1, 2)])
def test_training_workspace_follows_the_formula(net):
    """The LSTM layout against its restatement, and the same restatement with cell = 0 against the relu size, so the
    growth between the two is the one include/ctcb200.h and README.md state."""
    from _ctcb import lib
    for cell in (0, 1):
        cfg = _cfg(*net[:9], nt=net[9], cell=cell)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == _training_ws(*net, cell), cell


@pytest.mark.parametrize("net", [(41, 62, 512, 2, 1, 200, 32, 30, 0, 1), (13, 11, 70, 4, 2, 37, 5, 9, 1, 3)])
def test_lstm_activation_hooks(net):
    from _ctcb import lib
    cfg = _cfg(*net[:9], nt=net[9])
    relu = _cfg(*net[:9], nt=net[9], cell=0)
    off, w = ctypes.c_size_t(), ctypes.c_int32()
    tl, nt, H, uni = net[4], net[9], net[2], net[8]
    G = (1 if uni else 2) * 4 * H
    for layer in range(tl, tl + nt):
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), 0, layer, ctypes.byref(off), ctypes.byref(w)) == 0
        x = off.value
        assert w.value == G
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), 3, layer, ctypes.byref(off), ctypes.byref(w)) == 0
        assert (off.value, w.value) == (x, G)
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), 4, layer, ctypes.byref(off), ctypes.byref(w)) == 0
        assert w.value == H
        assert (lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), 5, layer, ctypes.byref(off), ctypes.byref(w)) == 0) \
            == (not uni)
    for what in (3, 4, 5):      # nothing of these kinds in a relu net
        assert lib.ctcb_brnn_activation_offset(ctypes.byref(relu), what, tl, ctypes.byref(off), ctypes.byref(w)) == -1


def test_cell_zero_is_the_config_without_the_member():
    """A config that never sets `cell` (ctypes zero-fills it) and one with cell = 0 report the same everything."""
    import _ctcb
    from _ctcb import lib
    for args in [(41, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0), (13, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 1, 2)]:
        a, b = _ctcb.BrnnConfig(*args), _ctcb.BrnnConfig(*args)
        b.cell = 0
        assert a.cell == 0
        assert _layout(a) == _layout(b)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(a)) == lib.ctcb_brnn_workspace_bytes(ctypes.byref(b))
        fa, fb = ctypes.c_size_t(), ctypes.c_size_t()
        assert (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(a), ctypes.byref(fa)), fa.value) == \
            (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(b), ctypes.byref(fb)), fb.value)


def test_lstm_sweep_entry_point_checks_its_arguments():
    from _ctcb import lib
    assert lib.ctcb_lstm_sweep_workspace_bytes(64, 8) == 4096 + 4096
    assert lib.ctcb_lstm_sweep_workspace_bytes(70, 3) == 4096 + (2 * 3 * 70 * 4 + 255) // 256 * 256
    assert lib.ctcb_lstm_sweep_workspace_bytes(0, 8) == 0
    # null pointers and bad sizes are refused before anything is enqueued
    assert lib.ctcb_lstm_sweep_f32(0, 4, 2, 64, None, None, None, None, None, None, None, None, None, None, None, 0,
                                   None) == -1
    assert "null pointer" in lib.ctcb_last_error().decode()


# ------------------------------------------------------------------------------------------- runNNet
def test_runnnet_cell_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).cell == "relu"
    cfg = runNNet.run_config(runNNet._parse(["--cell", "lstm"]))
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.trained_config(f).cell == "lstm"
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["cell"] == "lstm"       # resume keeps it
    old = dict(cfg)
    del old["cell"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.trained_config(f2).cell == "relu"                    # --test of a model from before the flag
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["cell"] == "relu"      # and its resume
