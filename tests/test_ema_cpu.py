"""CPU tests of the weight average (ctcb_ema_update_f32, SGD(emaDecay=d), runNNet --emaDecay): its float64 restatement
in tests/ema_oracle.py, the runNNet flags and configs, and the refusals that need no device."""
import inspect

import numpy as np
import pytest

import ema_oracle as oo


def _iterates(n=64, steps=40, seed=0):
    rng = np.random.RandomState(seed)
    return [(0.1 * rng.randn(n)).astype(np.float32) for _ in range(steps)]


def test_first_step_copies_w():
    w = _iterates(steps=1)[0]
    for a in (np.zeros_like(w), np.full_like(w, 7.0), -w):
        for t in (-3, 0, 1):
            assert np.array_equal(oo.ema_update(a, w, 0.999, t), w.astype(np.float64))
    assert oo.ema_decay(0.999, 1) == 0.0 and oo.ema_decay(0.999, 0) == 0.0


def test_below_the_warm_up_it_is_the_mean_of_the_iterates():
    """d = 0.99: 1 - 1/t < d up to t = 100, so every average of 40 steps is the running mean.  The restatement uses
    the decay rounded to float32 as the kernel does, so it equals the mean to float64 precision times that rounding."""
    ws = _iterates()
    a = np.zeros_like(ws[0], dtype=np.float64)
    for t, w in enumerate(ws, start=1):
        assert oo.ema_decay(0.99, t) == np.float64(np.float32(1.0 - 1.0 / t))
        a = oo.ema_update(a, w, 0.99, t)
        mean = np.mean(np.array(ws[:t], dtype=np.float64), axis=0)
        # d_t carries a relative rounding of at most 2^-24, on a - w of at most 2 max|w|, once per step
        assert np.abs(a - mean).max() <= t * 2.0 ** -23 * np.abs(np.array(ws[:t])).max(), t
    # with the decay's exact value the recurrence is the mean to float64 precision
    a = np.zeros_like(ws[0], dtype=np.float64)
    for t, w in enumerate(ws, start=1):
        a = w + (1.0 - 1.0 / t) * (a - w)
    assert np.abs(a - np.mean(np.array(ws, dtype=np.float64), axis=0)).max() < 1e-15


def test_above_the_warm_up_it_is_the_exponential_recurrence():
    d = 0.8                                     # 1 - 1/t >= d from t = 5
    ws = _iterates(steps=30, seed=1)
    a = np.zeros_like(ws[0])                  # the average is stored in float32 between steps, as on the device
    for t, w in enumerate(ws, start=1):
        prev = a.astype(np.float64)
        a64 = oo.ema_update(a, w, d, t)
        a = a64.astype(np.float32)
        if t >= 5:
            assert oo.ema_decay(d, t) == np.float64(np.float32(d))
            assert np.array_equal(a64, w.astype(np.float64) + np.float64(np.float32(d)) * (prev - w))
        else:
            assert oo.ema_decay(d, t) < np.float32(d)
    assert oo.ema_decay(d, 10 ** 6) == np.float64(np.float32(d))


def test_skipped_step_is_a_no_op():
    ws = _iterates(steps=2)
    a = ws[0]
    assert np.array_equal(oo.ema_update(a, ws[1], 0.9, 7, n_valid=0.0), a.astype(np.float64))
    assert not np.array_equal(oo.ema_update(a, ws[1], 0.9, 7, n_valid=3.0), a.astype(np.float64))


def test_ulps():
    x = np.array([1.0, -1.0, 0.0, -0.0, 1e-45], dtype=np.float32)
    assert oo.ulps(x, x).max() == 0
    assert oo.ulps(np.float32([0.0]), np.float32([-0.0]))[0] == 0
    assert oo.ulps(np.nextafter(x, np.float32(np.inf)), x).tolist() == [1, 1, 1, 1, 1]
    assert oo.ulps(np.float32([1e-45]), np.float32([-1e-45]))[0] == 2


def test_runnnet_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    flags = {f[0]: f for f in runNNet.FLAGS}
    assert flags["emaDecay"][1] is float and flags["emaDecay"][2] == 0.0 and flags["emaDecay"][3]
    assert flags["lastWeights"][1] is None and flags["lastWeights"][2] is False and flags["lastWeights"][3]
    assert runNNet._parse([]).emaDecay == 0.0 and runNNet._parse([]).lastWeights is False
    cfg = runNNet.run_config(runNNet._parse(["--emaDecay", "0.999"]))
    assert cfg["emaDecay"] == 0.999
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["emaDecay"] == 0.999
    assert runNNet.trained_config(f).emaDecay == 0.999
    old = {k: v for k, v in cfg.items() if k not in ("emaDecay", "lastWeights")}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["emaDecay"] == 0.0
    assert runNNet.trained_config(f2).emaDecay == 0.0
    assert runNNet.trained_config(f2).lastWeights is False


def test_sgd_default_is_off_and_refusals_come_first():
    """The decay is checked before the SGD touches the device or the net, so the refusals need neither."""
    import sgd
    assert inspect.signature(sgd.SGD.__init__).parameters["emaDecay"].default == 0.0
    for bad in (-0.1, 1.0, 1.5, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="emaDecay"):
            sgd.SGD(None, 10, emaDecay=bad)


def test_c_abi_refusals():
    """Host-side checks of ctcb_ema_update_f32: no launch happens, so no device is needed."""
    import ctypes
    from _ctcb import lib
    buf = (ctypes.c_float * 4)()
    step = (ctypes.c_int64 * 1)()
    p, s = ctypes.addressof(buf), ctypes.addressof(step)
    for d in (-0.5, 1.0, 2.0, float("nan"), float("inf")):
        assert lib.ctcb_ema_update_f32(p, p, 4, d, None, s, None) == -1, d
        assert b"decay" in lib.ctcb_last_error()
    for args in ((None, p, 4, 0.5, None, s), (p, None, 4, 0.5, None, s), (p, p, 4, 0.5, None, None)):
        assert lib.ctcb_ema_update_f32(*args, None) == -1, args
        assert b"null pointer" in lib.ctcb_last_error()
    for n in (0, -5):                                       # n <= 0: nothing to do, whatever the pointers
        assert lib.ctcb_ema_update_f32(None, None, n, 0.5, None, None, None) == 0
