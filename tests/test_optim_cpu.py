"""CPU tests of the adaptive optimisers (AdaGrad, Adam): the float64 rules of tests/optim_oracle.py on hand-computed
cases, AdaGrad's forgetting factor, the argument contract of ctcb_adagrad_step_f32 / ctcb_adam_step_f32 (checked on the
host before any launch), the params.pk state entry of every rule, and the runNNet flags.  No device is used."""
import ctypes
import math
import pickle

import numpy as np
import pytest

import optim_oracle as oo


# ------------------------------------------------------------------------------------------------ the oracle
def _close(a, b, tol=1e-12):
    return abs(float(np.asarray(a).reshape(-1)[0]) - b) <= tol * max(1.0, abs(b))


@pytest.mark.parametrize("t", [1, 2, 10])
@pytest.mark.parametrize("clip", [False, True])
def test_adagrad_by_hand(t, clip):
    """r is chosen so that gamma_t * r = 7 (gamma_t = t / (t + 100)); with g_c = 3, r' = 7 + 9 = 16 and
    w' = w - alpha * 3 / 4.  With the clip on, g = 9 and gnorm^2 = 36 over maxGNorm = 2 scale it by 1/3."""
    r = 7 * (t + 100) / t
    g, gnorm2, mx = (9.0, 36.0, 2.0) if clip else (3.0, 36.0, 100.0)
    out = oo.adagrad_step([1.0], [r], [g], 0.5, mx, gnorm2, t)
    assert _close(out["r"], 16.0)
    assert _close(out["w"], 1.0 - 0.5 * 3.0 / math.sqrt(16.0 + 1e-10))
    assert _close(out["S_r"], 16.0) and _close(out["S_w"], 1.0 + 0.375)


@pytest.mark.parametrize("t", [1, 2, 10])
@pytest.mark.parametrize("clip", [False, True])
def test_adam_by_hand(t, clip):
    """A gradient that has been g_c = 2 since step 1 leaves m = 2(1 - b1^(t-1)), v = 4(1 - b2^(t-1)) (exact in float32
    for b1 = 1/2, b2 = 3/4), so the bias-corrected moments are exactly g_c and g_c^2 and the step is
    alpha * 2 / (2 + eps).  With the clip on, g = 8 and gnorm^2 = 16 over maxGNorm = 1 scale it by 1/4."""
    b1, b2, eps, alpha = 0.5, 0.75, 1e-8, 0.5
    m0, v0 = 2.0 * (1 - b1 ** (t - 1)), 4.0 * (1 - b2 ** (t - 1))
    assert np.float32(m0) == m0 and np.float32(v0) == v0
    g, gnorm2, mx = (8.0, 16.0, 1.0) if clip else (2.0, 16.0, 100.0)
    out = oo.adam_step([1.0], [m0], [v0], [g], alpha, b1, b2, eps, mx, gnorm2, t)
    assert _close(out["m"], 2.0 * (1 - b1 ** t)) and _close(out["v"], 4.0 * (1 - b2 ** t))
    assert _close(out["w"], 1.0 - alpha * 2.0 / (2.0 + eps))
    # and the rule itself, written out for this t
    m1, v1 = b1 * m0 + (1 - b1) * 2.0, b2 * v0 + (1 - b2) * 4.0
    assert _close(out["w"], 1.0 - alpha * (m1 / (1 - b1 ** t)) / (math.sqrt(v1 / (1 - b2 ** t)) + eps))


def test_adam_first_step_moves_each_element_by_about_alpha():
    """At t = 1 from zero moments every element with |g| >> eps moves by alpha * sign(g), whatever its size."""
    g = np.array([1e-3, -2.0, 50.0, -1e-6], dtype=np.float32)
    z = np.zeros(4, np.float32)
    out = oo.adam_step(z, z, z, g, 1e-2, 0.9, 0.999, 1e-8, 1e9, 1.0, 1)
    assert np.allclose(out["w"], -1e-2 * np.sign(g), rtol=1e-2)


def test_skipped_step_changes_nothing_and_t_below_one_is_one():
    rng = np.random.RandomState(0)
    w, s1, s2, g = (rng.randn(5).astype(np.float32) for _ in range(4))
    s2 = np.abs(s2)
    a = oo.adagrad_step(w, np.abs(s1), g, 0.1, 1.0, 4.0, 3, n_valid=0.0)
    assert np.array_equal(a["w"], w) and np.array_equal(a["r"], np.abs(s1))
    b = oo.adam_step(w, s1, s2, g, 0.1, 0.9, 0.999, 1e-8, 1.0, 4.0, 3, n_valid=0.0)
    assert np.array_equal(b["w"], w) and np.array_equal(b["m"], s1) and np.array_equal(b["v"], s2)
    assert not np.array_equal(oo.adam_step(w, s1, s2, g, 0.1, 0.9, 0.999, 1e-8, 1.0, 4.0, 3, n_valid=2.0)["w"], w)
    for t in (0, -1, -2 ** 40):
        assert oo.step_number(t) == 1
        for k in ("w", "r"):
            assert np.array_equal(oo.adagrad_step(w, np.abs(s1), g, 0.1, 1.0, 4.0, t)[k],
                                  oo.adagrad_step(w, np.abs(s1), g, 0.1, 1.0, 4.0, 1)[k])
        for k in ("w", "m", "v"):
            assert np.array_equal(oo.adam_step(w, s1, s2, g, 0.1, 0.9, 0.999, 1e-8, 1.0, 4.0, t)[k],
                                  oo.adam_step(w, s1, s2, g, 0.1, 0.9, 0.999, 1e-8, 1.0, 4.0, 1)[k])


def test_adagrad_forgetting_factor():
    """gamma_t = 1 - 1/(0.01 t + 1) = t / (t + 100): 1/101 at t = 1, 1/2 at t = 100, increasing towards 1."""
    gam = [oo.adagrad_gamma(t) for t in range(1, 20001)]
    assert abs(gam[0] - 1 / 101) < 1e-16 and abs(gam[99] - 0.5) < 1e-16 and abs(gam[9] - 1 / 11) < 1e-16
    assert all(a < b for a, b in zip(gam, gam[1:]))
    assert 1 - gam[-1] < 0.005 and oo.adagrad_gamma(2 ** 40) < 1.0
    assert oo.adagrad_gamma(0) == oo.adagrad_gamma(1)


def test_clip_scale():
    assert oo.clip_scale(4.0, 5.0) == 1.0 and oo.clip_scale(0.0, 5.0) == 1.0
    assert oo.clip_scale(100.0, 5.0) == 0.5
    assert oo.clip_scale(25.0, 5.0) == 1.0            # at the threshold: no clip, as the Nesterov kernel decides


# ------------------------------------------------------------------------------------------------ C ABI
def test_argument_contract_is_checked_before_any_launch():
    from _ctcb import lib
    buf = (ctypes.c_float * 8)()
    p = ctypes.addressof(buf)
    step = ctypes.c_int64(1)
    sp = ctypes.addressof(step)
    nan, inf = float("nan"), float("inf")

    def adagrad(w=p, r=p, g=p, n=8, alpha=0.1, gnorm2=p, step=sp):
        return lib.ctcb_adagrad_step_f32(w, r, g, n, alpha, 1.0, gnorm2, None, step, None)

    def adam(w=p, m=p, v=p, g=p, n=8, alpha=0.1, b1=0.9, b2=0.999, eps=1e-8, gnorm2=p, step=sp):
        return lib.ctcb_adam_step_f32(w, m, v, g, n, alpha, b1, b2, eps, 1.0, gnorm2, None, step, None)

    n0 = lib.ctcb_launch_count()
    for n in (0, -1):                                   # n <= 0: a no-op, whatever the rest
        assert adagrad(w=None, n=n, alpha=nan) == 0
        assert adam(w=None, n=n, b1=2.0) == 0
    for k in ("w", "r", "g", "gnorm2", "step"):
        assert adagrad(**{k: None}) == -1, k
        assert b"ctcb_adagrad_step_f32" in lib.ctcb_last_error()
    for k in ("w", "m", "v", "g", "gnorm2", "step"):
        assert adam(**{k: None}) == -1, k
    for a in (nan, inf, -inf, -1e-6):
        assert adagrad(alpha=a) == -1 and b"alpha" in lib.ctcb_last_error()
        assert adam(alpha=a) == -1 and b"alpha" in lib.ctcb_last_error()
    for b in (1.0, 1.5, -0.1, nan, inf):
        assert adam(b1=b) == -1 and b"beta" in lib.ctcb_last_error()
        assert adam(b2=b) == -1 and b"beta" in lib.ctcb_last_error()
    for e in (0.0, -1e-8, nan, inf):
        assert adam(eps=e) == -1 and b"eps" in lib.ctcb_last_error()
    assert lib.ctcb_launch_count() == n0


def test_sgd_refuses_unknown_rules_and_bad_adam_arguments():
    """Checked before any device is touched (model None is never read)."""
    import sgd
    for name in ("adadelta", "rmsprop", "sgd", "Adam", ""):
        with pytest.raises(ValueError, match="adagrad, adam, nesterov"):
            sgd.SGD(None, 10, optimizer=name)
    for kw in (dict(beta1=1.0), dict(beta2=-0.5), dict(beta1=float("nan")), dict(epsilon=0.0),
               dict(epsilon=float("inf"))):
        with pytest.raises(ValueError):
            sgd.SGD(None, 10, optimizer="adam", **kw)


# ------------------------------------------------------------------------------------------------ checkpoint
def _pairs(seed, shapes=((4, 3), (4, 1), (2, 4), (2, 1))):
    rng = np.random.RandomState(seed)
    arr = [rng.randn(*s).astype(np.float32) for s in shapes]
    return [[arr[i], arr[i + 1]] for i in range(0, len(arr), 2)]


@pytest.mark.parametrize("rule", ["nesterov", "adagrad", "adam"])
def test_checkpoint_state_entry(rule):
    """The first pickle stays [it, costt, expcost, state] (plot_results.py and the reference's fromFile unpack four
    values); Nesterov's state is the reference's list of velocity pairs; every rule reads back what it wrote."""
    import sgd
    names = sgd.OPTIMIZERS[rule]
    pairs = {name: _pairs(k) for k, name in enumerate(names)}
    blob = pickle.dumps([7, [1.5, 1.25], [1.5, 1.4], sgd.pack_state(rule, pairs)])
    it, costt, expcost, state = pickle.loads(blob)
    assert it == 7 and costt == [1.5, 1.25] and expcost == [1.5, 1.4]
    if rule == "nesterov":
        assert isinstance(state, list) and len(state) == 2
    else:
        assert state["optimizer"] == rule and sorted(state) == sorted(("optimizer",) + names)
    back = sgd.unpack_state(rule, state)
    assert sorted(back) == sorted(names)
    for name in names:
        for (a, b), (x, y) in zip(back[name], pairs[name]):
            assert np.array_equal(a, x) and np.array_equal(b, y)


def test_nesterov_entry_is_the_reference_format():
    import sgd
    pairs = _pairs(3)
    assert sgd.pack_state("nesterov", {"velocity": pairs}) is pairs


@pytest.mark.parametrize("saved,loading", [("nesterov", "adam"), ("adam", "nesterov"), ("adagrad", "adam"),
                                           ("adam", "adagrad"), ("nesterov", "adagrad"), ("adagrad", "nesterov")])
def test_checkpoint_of_another_rule_is_refused(saved, loading):
    import sgd
    state = sgd.pack_state(saved, {name: _pairs(1) for name in sgd.OPTIMIZERS[saved]})
    with pytest.raises(ValueError) as e:
        sgd.unpack_state(loading, pickle.loads(pickle.dumps(state)))
    assert repr(saved) in str(e.value) and repr(loading) in str(e.value)


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_optimizer_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    d = runNNet._parse([])
    assert (d.optimizer, d.beta1, d.beta2, d.epsilon) == ("nesterov", 0.9, 0.999, 1e-8)
    cfg = runNNet.run_config(runNNet._parse(["--optimizer", "adam", "--beta1", "0.8", "--beta2", "0.99",
                                             "--epsilon", "1e-6"]))
    assert (cfg["optimizer"], cfg["beta1"], cfg["beta2"], cfg["epsilon"]) == ("adam", 0.8, 0.99, 1e-6)
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f, "--optimizer", "adagrad"]))
    assert (back["optimizer"], back["beta1"], back["beta2"], back["epsilon"]) == ("adam", 0.8, 0.99, 1e-6)
    old = dict(cfg)
    for k in ("optimizer", "beta1", "beta2", "epsilon"):
        del old[k]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    back = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))       # a run from before the flags
    assert (back["optimizer"], back["beta1"], back["beta2"], back["epsilon"]) == ("nesterov", 0.9, 0.999, 1e-8)
    assert runNNet.trained_config(f2).optimizer == "nesterov"
