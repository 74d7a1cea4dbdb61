"""CPU tests of the Gaussian weight noise: the NumPy restatement (tests/weight_noise_oracle.py) against a plain loop over
every element, its law, its counters against the other two draws of a seed, and the C ABI's config, setter and
workspace contract (no device work)."""
import ctypes
import math

import numpy as np
import pytest
from scipy import stats

import weight_noise_oracle as wno
from net_oracle import philox4x32_10


def _loop_terms(sigma, seed, step, lo, hi):
    """The rule of include/ctcb200.h spelt out one element at a time, from the Philox blocks alone."""
    out = []
    for e in range(lo, hi):
        q, j = e // 4, e % 4
        ctr = np.array([[step % 2 ** 32, q % 2 ** 32, 1, 0]], dtype=np.uint64)
        r = [int(x) for x in philox4x32_10(ctr, (seed % 2 ** 32, seed >> 32))[0]]
        a, b = (r[0], r[1]) if j < 2 else (r[2], r[3])
        u1, u2 = (a + 1) * 2.0 ** -32, b * 2.0 ** -32
        rho = math.sqrt(-2.0 * math.log(u1))
        z = rho * (math.cos(2 * math.pi * u2) if j % 2 == 0 else math.sin(2 * math.pi * u2))
        out.append(np.float32(float(np.float32(sigma)) * z))
    return np.array(out, dtype=np.float32)


def _ulps(a, b):
    a, b = a.astype(np.float32), b.astype(np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


LOOP_CASES = [
    # sigma, seed, step, lo, hi
    (0.075, 33, 0, 0, 203),
    (1.0, 2 ** 40 + 5, 2 ** 33 + 7, 4 * (2 ** 32 - 8), 4 * (2 ** 32 + 9) + 3),      # q crosses 2^32: it wraps
    (0.5, 7, 12, 1024, 1030),
    (3e-3, 2 ** 64 - 1, 2 ** 63 - 1, 40, 41),
]


@pytest.mark.parametrize("case", range(len(LOOP_CASES)))
def test_restatement_equals_a_plain_loop(case):
    sigma, seed, step, lo, hi = LOOP_CASES[case]
    want = _loop_terms(sigma, seed, step, lo, hi)
    got = wno.terms(sigma, seed, step, lo, hi)
    d = _ulps(got, want)
    # math.cos(2 pi u2) loses relative accuracy only within ~1e-9 of its zeros; none of these elements is near one
    assert d.max() <= 1, d.max()
    assert (d == 0).mean() > 0.95


def test_quad_words_and_seed_halves_change_the_draws():
    base = wno.draws(5, 3, [7, 8])
    for other in (wno.draws(5, 4, [7, 8]), wno.draws(5, 3, [9, 10]), wno.draws(5 + 2 ** 32, 3, [7, 8])):
        assert not np.array_equal(base, other)
    assert np.array_equal(base, wno.draws(5, 3 + 2 ** 32, [7 + 2 ** 32, 8 + 2 ** 32]))     # step and q enter mod 2^32
    # one block per quad: elements 0, 1 share (r0, r1), elements 2, 3 share (r2, r3), and the pairs are orthogonal
    z = wno.normals(9, 1, 0, 8)
    r = wno.draws(9, 1, [0, 1])
    rho = np.sqrt(-2 * np.log((r[:, [0, 2]].astype(np.float64) + 1) * 2.0 ** -32)).reshape(-1)
    assert np.allclose(np.hypot(z[0::2], z[1::2]), rho, rtol=1e-14)


def test_the_reduced_sincos_is_the_circle():
    b = np.array([0, 1, 2 ** 30, 2 ** 30 + 1, 2 ** 31, 3 * 2 ** 30, 2 ** 32 - 1, 12345678, 2 ** 29 + 7], dtype=np.float64)
    s, c = wno.sincos_2pi(b * 2.0 ** -32)
    assert np.allclose(s, np.sin(2 * np.pi * b * 2.0 ** -32), atol=1e-15)
    assert np.allclose(c, np.cos(2 * np.pi * b * 2.0 ** -32), atol=1e-15)
    assert s[0] == 0.0 and c[0] == 1.0 and c[2] == 0.0 and s[4] == 0.0 and c[5] == 0.0
    # near a zero the relative accuracy stays: sin(2 pi 2^-32) = 2 pi 2^-32 (1 - ...)
    assert abs(s[1] / (2 * np.pi * 2.0 ** -32) - 1) < 1e-15


def test_draws_are_standard_normal():
    """z ~ N(0, 1): a Kolmogorov-Smirnov test over 2^20 draws of one step, and one over the first elements of many
    steps (the noise moves with the counter)."""
    z = wno.normals(33, 5, 0, 2 ** 20)
    assert np.isfinite(z).all()
    assert stats.kstest(z, "norm").pvalue > 1e-3
    assert abs(z.mean()) < 5e-3 and abs(z.var() - 1) < 5e-3
    # the two members of a Box-Muller pair are uncorrelated
    assert abs(np.corrcoef(z[0::2], z[1::2])[0, 1]) < 5e-3
    across = np.array([wno.normals(33, s, 0, 4) for s in range(4096)]).reshape(-1)
    assert stats.kstest(across, "norm").pvalue > 1e-3


def test_apply_noises_only_the_ranges_and_copies_the_rest_bit_for_bit():
    rng = np.random.RandomState(1)
    p = rng.randn(64).astype(np.float32)
    p[10] = -0.0
    p[30] = np.nan
    ranges = [(0, 9), (12, 30), (40, 41)]
    out = wno.apply(p, ranges, 0.1, 3, 4)
    inside = np.zeros(64, dtype=bool)
    for lo, hi in ranges:
        inside[lo:hi] = True
        assert np.array_equal(out[lo:hi], p[lo:hi] + wno.terms(0.1, 3, 4, lo, hi))
    assert np.array_equal(out.view(np.uint32)[~inside], p.view(np.uint32)[~inside])
    assert (out[inside] != p[inside]).all()
    # an element's noise depends on its offset alone, not on the range it lies in
    assert np.array_equal(wno.terms(0.1, 3, 4, 12, 30)[4:], wno.terms(0.1, 3, 4, 16, 30))


def test_counters_never_meet_dropout_or_the_input_masks():
    """This rule's counters are (s, q, 1, 0).  Dropout's are (s, g, t, (layer << 24) | j / 4) with layer >= 1, so their
    fourth word is >= 2^24; SpecAugment's are (s, g, 0, k), third word 0.  Under any seed and step none of the three
    sets meets another: checked on the words and on sampled counters of each."""
    steps = [0, 1, 7, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3]
    ours = np.concatenate([wno.counters(s, np.array([0, 1, 5, 2 ** 24, 2 ** 32 - 1, 2 ** 32 + 2, 2 ** 40],
                                                    dtype=np.uint64)) for s in steps])
    assert (ours[:, 2] == 1).all() and (ours[:, 3] == 0).all()
    drop = []
    for s in steps:
        for layer in (1, 2, 64):
            for g, t, q in ((0, 0, 0), (1, 1, 0), (0, 1, 3), (5, 0, 1)):
                drop.append((s & wno.M32, g, t, (layer << 24) | q))
    masks = [(s & wno.M32, g, 0, k) for s in steps for g in (0, 1, 5) for k in (0, 1, 127)]
    drop, masks = np.array(drop, dtype=np.uint64), np.array(masks, dtype=np.uint64)
    assert (drop[:, 3] >= 2 ** 24).all() and (masks[:, 2] == 0).all()
    as_set = lambda a: set(map(tuple, a.tolist()))
    assert not as_set(ours) & as_set(drop) and not as_set(ours) & as_set(masks)


# ------------------------------------------------------------------------------------------------------- C ABI
def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


CFG_CASES = {
    "bi_relu": dict(),
    "uni_k2": dict(unidirectional=1, temporalLayer=1, numTemporal=2),
    "dnn": dict(temporalLayer=0),
    "lstm_peephole_ln": dict(cell=1, peephole=1, layerNorm=1),
    "subsample": dict(subsample=2, subsampleLayer=2, layerSize=63),
    "masks": dict(maskFeatDim=41),
}


@pytest.mark.parametrize("name", list(CFG_CASES))
def test_workspace_grows_by_exactly_the_copy(name):
    from _ctcb import lib
    off = _cfg(**CFG_CASES[name])
    assert off.weightNoise == 0          # an initialiser without the member keeps its meaning
    on = _cfg(weightNoise=1, **CFG_CASES[name])
    base = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    P = lib.ctcb_brnn_param_count(ctypes.byref(off))
    assert base > 0 and P > 0
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(on)) == base + (4 * P + 255) // 256 * 256
    assert lib.ctcb_brnn_param_count(ctypes.byref(on)) == P
    assert lib.ctcb_brnn_num_tensors(ctypes.byref(on)) == lib.ctcb_brnn_num_tensors(ctypes.byref(off))
    assert (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(on), None)
            == lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), None))
    assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(on)) == lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))
    for what, layer in ((0, 1), (0, 4), (7, 1), (7, 4), (1, 2)):
        a, b = ctypes.c_size_t(), ctypes.c_size_t()
        ra = lib.ctcb_brnn_activation_offset(ctypes.byref(off), what, layer, ctypes.byref(a), None)
        rb = lib.ctcb_brnn_activation_offset(ctypes.byref(on), what, layer, ctypes.byref(b), None)
        assert ra == rb and a.value == b.value, (what, layer)
    # the noised ranges: the matrices only, each quad-aligned, ascending, inside the vector
    ranges = wno.cfg_ranges(on)
    assert all(lo % 4 == 0 and lo < hi for lo, hi in ranges)
    assert all(a[1] < b[0] for a, b in zip(ranges, ranges[1:])) and ranges[-1][1] <= P


def test_config_refusals():
    from _ctcb import lib
    for v in (-1, 2, 7):
        cfg = _cfg(weightNoise=v)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, v
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, v
        msg = lib.ctcb_last_error()
        assert b"weightNoise %d" % v in msg and b"neither 0" in msg, msg


def test_set_weight_noise_argument_contract():
    from _ctcb import lib
    step = ctypes.c_int64(0)     # the setter only stores the pointer: a host address does for the contract
    sp = ctypes.addressof(step)
    h, h0 = ctypes.c_void_p(), ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg(weightNoise=1)), ctypes.byref(h)) == 0
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg()), ctypes.byref(h0)) == 0
    n0 = lib.ctcb_launch_count()
    try:
        set_ = lib.ctcb_brnn_set_weight_noise
        assert set_(h, 0.075, 33, sp) == 0
        assert set_(h, 1e30, 2 ** 64 - 1, sp) == 0
        assert set_(h, 0.0, 0, None) == 0                       # sigma 0: off, no counter needed
        for bad in (-0.1, -1e-30, float("nan"), float("inf"), float("-inf")):
            assert set_(h, bad, 1, sp) == -1, bad
            msg = lib.ctcb_last_error()
            assert b"ctcb_brnn_set_weight_noise" in msg and b"not a finite value >= 0" in msg, msg
        assert set_(h, 0.1, 1, None) == -1 and b"step counter" in lib.ctcb_last_error()
        assert set_(h0, 0.1, 1, sp) == -1 and b"weightNoise = 1" in lib.ctcb_last_error()
        assert set_(h0, 0.0, 1, None) == 0                      # no copy, no noise: nothing to refuse
        assert set_(None, 0.0, 1, sp) == -1 and b"null handle" in lib.ctcb_last_error()
        # the pass alone refuses null pointers and overlapping arrays before any device work
        P = lib.ctcb_brnn_param_count(ctypes.byref(_cfg(weightNoise=1)))
        x = 1 << 20
        f = lib.ctcb_brnn_weight_noise_f32
        for args in ((None, x, x + 8 * P), (h, None, x), (h, x, None), (h, x, x + 4 * P - 4), (h, x + 4, x),
                     (h, x, x)):
            assert f(*args, None) == -1, args
            assert b"ctcb_brnn_weight_noise_f32" in lib.ctcb_last_error()
        assert b"overlaps" in lib.ctcb_last_error()
    finally:
        lib.ctcb_brnn_destroy(h)
        lib.ctcb_brnn_destroy(h0)
    assert lib.ctcb_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_weight_noise_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).weightNoise == 0.0
    assert any(f[0] == "weightNoise" and f[3] for f in runNNet.FLAGS)      # it has a help text
    cfg = runNNet.run_config(runNNet._parse(["--weightNoise", "0.075"]))
    assert cfg["weightNoise"] == 0.075
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["weightNoise"] == 0.075
    old = {k: v for k, v in cfg.items() if k != "weightNoise"}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["weightNoise"] == 0.0
    assert runNNet.trained_config(f2).weightNoise == 0.0
