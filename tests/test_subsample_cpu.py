"""CPU tests of frame subsampling (ctcb_brnn_config.subsample = k at map subsampleLayer = L): subsampling off is the net
without the members (every config answer over 25,600 configs against the build before them), the config contract
(refusals, W_L's shape, the workspace), the host admission rule at ceil(T / k), and runNNet's flags (the float64
restatement of the net is tested in tests/test_net_oracle_cpu.py)."""
import ctypes
import os

import numpy as np
import pytest

import config_matrix

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cfg(D, K, H, N, tl, T, B, L=9, uni=0, nt=1, cell=0, ln=0, k=2, sl=1):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, T, B, L, 0.0, 20.0, uni, nt, cell, ln, k, sl)


def _shapes(cfg):
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


# ------------------------------------------------------------------------------------------- off is today's net
@pytest.mark.parametrize("k, sl", [(0, 0), (1, 3), (0, 99), (1, -4)])
def test_subsampling_off_answers_every_config_query_as_before(k, sl):
    """subsample = 0 or 1 (subsampleLayer ignored) gives, for every config of the matrix, the parameter count, the tensor
    table, both workspace sizes and flag offsets, the activation offsets and create's return code of the build before
    the members existed.  Some answers depend on the device the planners see (workspace sizes, create's checks), so
    there is one fixture for a machine without a device and one for an H100 SXM; another device is skipped."""
    import _ctcb
    from _ctcb import lib
    golden = _golden()
    if golden is None:
        pytest.skip("the fixtures are those of no device and of an H100 SXM (sm_90, 132 SMs), not of this device")
    want = np.load(golden)["digests"]
    assert len(want) == len(config_matrix.MATRIX)
    config_matrix.bind(lib, _ctcb.BrnnConfig)
    got = np.array([config_matrix.digest(config_matrix.answers(lib, config_matrix.config(_ctcb.BrnnConfig, e, k, sl)))
                    for e in config_matrix.MATRIX], dtype=np.int64)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [config_matrix.MATRIX[i] for i in bad[:5]]


# ------------------------------------------------------------------------------------------- the config contract
def test_invalid_subsampling_is_refused_with_a_message():
    from _ctcb import lib
    h = ctypes.c_void_p()
    for k, sl, text in ((-1, 1, "subsample -1 is negative"), (-5, 0, "subsample -5"),
                        (2, 0, "subsampleLayer 0 is not one of the affine maps 1..4"),
                        (3, 5, "subsampleLayer 5 is not one of the affine maps 1..4 (numLayers + 1) that subsample 3")):
        cfg = _cfg(13, 11, 64, 3, 2, 60, 8, k=k, sl=sl)
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
        assert text in lib.ctcb_last_error().decode(), lib.ctcb_last_error()
        assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0
        assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == 0
    for sl in (1, 2, 3, 4):
        cfg = _cfg(13, 11, 64, 3, 2, 60, 8, k=2, sl=sl)
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
        lib.ctcb_brnn_destroy(h)


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("sl", [1, 2, 3, 4])
def test_only_w_l_widens(k, sl):
    """W_L is rows x k n; every tensor keeps its place in the order, the offsets behind W_L move by its growth."""
    D, K, H = 13, 11, 64
    off, on = _shapes(_cfg(D, K, H, 3, 2, 60, 8, k=1)), _shapes(_cfg(D, K, H, 3, 2, 60, 8, k=k, sl=sl))
    assert len(on) == len(off)
    n = D if sl == 1 else H
    rows = off[2 * (sl - 1)][1]
    growth = (rows * k * n + 3) // 4 * 4 - (rows * n + 3) // 4 * 4
    for t, ((o0, r0, c0), (o1, r1, c1)) in enumerate(zip(off, on)):
        assert r1 == r0
        assert c1 == (k * c0 if t == 2 * (sl - 1) else c0)
        assert o1 == o0 + (0 if t <= 2 * (sl - 1) else growth)
    assert on[2 * (sl - 1)][2] == k * n


def _ws(cfg):
    from _ctcb import lib
    return lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg))


def test_forward_only_calls_fit_in_the_training_workspace():
    """A forward-only call runs in the training workspace (nnets.brnnet.NNet.forwardBatch on a training net): for every
    valid config of the matrix at k = 2, 3, 4 and every L, the forward workspace is no larger than the training one.
    The forward buffers above L hold R' rows, as the training buffers do."""
    import _ctcb
    from _ctcb import lib
    n = 0
    for e in config_matrix.MATRIX:
        for k in (2, 3, 4):
            for sl in range(1, e[3] + 2):
                cfg = config_matrix.config(_ctcb.BrnnConfig, e, k, sl)
                train = lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg))
                if train:
                    n += 1
                    assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) <= train, (e, k, sl)
    assert n > 150000
    # C2 with LSTM layers from map 1, and C3 at k = 4 from map 1
    for net in ((41, 62, 512, 2, 1, 200, 32, 30, 0, 1, 1, 0, 2, 1), (41, 32, 1024, 3, 2, 800, 128, 100, 0, 1, 0, 0, 4, 1)):
        cfg = _cfg(*net)
        assert 0 < lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) <= _ws(cfg)


def test_workspace_above_the_subsampling_point_shrinks():
    """C3 shape (3 layers of 1024, temporal layer 2, 800 x 128): k = 2 from map 2 sizes X_2.., D_2.., For / Back, the
    pairs and the CTC area for 400 x 128 rows and adds S, dS (each 51200 x 2048 floats) and T'."""
    from _ctcb import lib
    al = lambda x: (x + 255) // 256 * 256     # noqa: E731
    base, sub = _cfg(41, 32, 1024, 3, 2, 800, 128, L=100, k=1), _cfg(41, 32, 1024, 3, 2, 800, 128, L=100, k=2, sl=2)
    assert _ws(sub) < _ws(base)
    o, w = ctypes.c_size_t(), ctypes.c_int32()
    assert lib.ctcb_brnn_activation_offset(ctypes.byref(sub), 6, 0, ctypes.byref(o), ctypes.byref(w)) == 0
    assert w.value == 2 * 1024
    assert _ws(sub) - o.value == 2 * al(51200 * 2048 * 4) + al(128 * 4)
    assert lib.ctcb_brnn_activation_offset(ctypes.byref(base), 6, 0, ctypes.byref(o), ctypes.byref(w)) == -1
    # X_1 keeps 102400 rows, X_2 has 51200
    x1, x2 = ctypes.c_size_t(), ctypes.c_size_t()
    lib.ctcb_brnn_activation_offset(ctypes.byref(sub), 0, 1, ctypes.byref(x1), None)
    lib.ctcb_brnn_activation_offset(ctypes.byref(sub), 0, 2, ctypes.byref(x2), None)
    assert x2.value - x1.value == al(102400 * 1024 * 4)
    # L = 1: no dS, every map at the reduced rate
    one = _cfg(41, 32, 1024, 3, 2, 800, 128, L=100, k=2, sl=1)
    assert lib.ctcb_brnn_activation_offset(ctypes.byref(one), 6, 0, ctypes.byref(o), ctypes.byref(w)) == 0
    assert w.value == 2 * 41 and _ws(one) - o.value == al(51200 * 82 * 4) + al(128 * 4)


# ------------------------------------------------------------------------------------------- host side
def test_admission_compares_ceil_t_over_k_with_the_labels():
    import parallel
    dd = {"a": np.zeros((3, 10)), "b": np.zeros((3, 9)), "c": np.zeros((3, 7)), "d": np.zeros((3, 30))}
    alis = {"a": list(range(4)), "b": list(range(3)), "c": list(range(3)), "d": list(range(11))}
    keys = ["a", "b", "c", "d"]
    assert parallel.select_step_utterances(dd, alis, keys, 60, 0, 1) == keys
    logs = []
    # k = 3: a 4 frames >= 4, b 3 >= 3, c 3 >= 3, d 10 < 11
    assert parallel.select_step_utterances(dd, alis, keys, 60, 0, 1, log=logs.append, subsample=3) == ["a", "b", "c"]
    assert len(logs) == 1 and "Utterance length 10, Num Labels 11" in logs[0]
    # k = 4: a 3 < 4, b 3 >= 3, c 2 < 3, d 8 < 11
    assert parallel.select_step_utterances(dd, alis, keys, 60, 0, 1, subsample=4) == ["b"]
    assert parallel.select_step_utterances(dd, alis, keys, 60, 0, 1, subsample=1) == keys


def test_runnnet_subsample_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    o = runNNet._parse([])
    assert (o.subsample, o.subsampleLayer) == (1, 1)
    o = runNNet._parse(["--subsample", "3", "--subsampleLayer", "2"])
    assert (o.subsample, o.subsampleLayer) == (3, 2)
    cfg = runNNet.run_config(o)
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    t = runNNet.trained_config(f)
    assert (t.subsample, t.subsampleLayer) == (3, 2)                                       # --test rebuilds it
    r = runNNet.run_config(runNNet._parse(["--cfg_file", f]))
    assert (r["subsample"], r["subsampleLayer"]) == (3, 2)                                 # resume keeps it
    old = dict(cfg)
    del old["subsample"], old["subsampleLayer"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    t = runNNet.trained_config(f2)
    assert (t.subsample, t.subsampleLayer) == (1, 1)                                       # a model from before
    r = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))
    assert (r["subsample"], r["subsampleLayer"]) == (1, 1)


def test_entry_points_check_their_arguments():
    from _ctcb import lib
    assert lib.ctcb_frame_stack_f32(None, None, 4, 2, 8, 2, None, None, None) == -1
    assert "null pointer" in lib.ctcb_last_error().decode()
    assert lib.ctcb_frame_stack_f32(None, None, 4, 2, 8, 0, None, None, None) == -1
    assert "k = 0" in lib.ctcb_last_error().decode()
    assert lib.ctcb_frame_unstack_f32(None, None, 0, 2, 8, 2, None, None) == -1
    assert "Tmax = 0" in lib.ctcb_last_error().decode()
