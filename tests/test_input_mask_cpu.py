"""CPU tests of the SpecAugment input masks: the NumPy restatement (tests/input_mask_oracle.py) against a plain loop
over every element, its edges and laws, and the C ABI's config, setter and workspace contract (no device work)."""
import ctypes

import numpy as np
import pytest
from scipy import stats

import input_mask_oracle as imo


def _loop_mask(lens, Tmax, D, nu, mF, F, mT, Tw, p, seed, step, first=0, stride=1):
    """The policy of include/ctcb200.h spelt out one element at a time, from the Philox blocks alone."""
    c, h = D // nu, (D // nu - 1) // 2
    out = np.zeros((Tmax, len(lens), D), dtype=bool)
    for u, Tu in enumerate(lens):
        r = imo.draws(seed, step, first + stride * u, mF + mT)
        fb, tb = [], []
        for k in range(mF + mT):
            r0, r1 = int(r[k, 0]), int(r[k, 1])
            if k < mF:
                w = r0 * (F + 1) // 2 ** 32
                f0 = r1 * (nu - w + 1) // 2 ** 32
                fb.append(range(f0, f0 + w))
            else:
                W = min(Tw, int(np.floor(float(p) * Tu)))
                w = r0 * (W + 1) // 2 ** 32
                t0 = r1 * (Tu - w + 1) // 2 ** 32
                tb.append(range(t0, t0 + w))
        for t in range(min(Tu, Tmax)):
            for j in range(c):
                f = min(max(t + j - h, 0), Tu - 1)
                for b in range(nu):
                    out[t, u, j * nu + b] = any(b in x for x in fb) or any(f in x for x in tb)
    return out


LOOP_CASES = [
    # lens, nu, c, mF, F, mT, Tw, p, seed, step, first, stride
    ([9, 4, 7], 5, 3, 2, 3, 2, 4, 0.5, 33, 3, 0, 1),
    ([12, 1, 6, 2], 4, 5, 3, 4, 3, 6, 1.0, 2 ** 40 + 5, 2 ** 33 + 7, 7, 3),
    ([10, 10], 7, 1, 1, 7, 4, 10, 0.3, 5, 0, 70000, 2),
    ([3, 8], 3, 7, 64, 2, 64, 3, 1.0, 11, 9, 0, 1),
]


@pytest.mark.parametrize("case", range(len(LOOP_CASES)))
def test_restatement_equals_a_plain_loop(case):
    lens, nu, c, mF, F, mT, Tw, p, seed, step, first, stride = LOOP_CASES[case]
    Tmax = max(lens) + 2          # padded rows too
    args = (lens, Tmax, nu * c, nu, mF, F, mT, Tw, p, seed, step, first, stride)
    want = _loop_mask(*args)
    got = imo.batch_mask(*args)
    assert np.array_equal(got, want)
    assert got.any() and not got.all()


def test_apply_zeroes_only_masked_elements_and_copies_the_rest_bit_for_bit():
    rng = np.random.RandomState(1)
    x = rng.randn(6, 2, 15).astype(np.float32)
    x[0, 0, 0] = -0.0
    x[5, 1, 3] = np.nan
    m = imo.batch_mask([4, 6], 6, 15, 5, 2, 5, 2, 3, 1.0, 3, 1)
    y = imo.apply(x, m)
    assert np.array_equal(y.view(np.uint32)[~m], x.view(np.uint32)[~m])
    assert (y.view(np.uint32)[m] == 0).all()         # +0.0, not -0.0
    assert not m[4:, 0].any()                         # padding rows of the 4-frame utterance are copied


# ------------------------------------------------------------------------------------------------------- edges
def test_one_frame_utterance():
    """T_u = 1: W <= 1 and every slot holds frame 0, so a time mask of width 1 zeroes the whole row."""
    widths = set()
    for step in range(40):
        f, t = imo.bands(3, step, 0, 5, 1, 0, 0, 1, 10, 1.0)
        (a, b), = t
        assert (a, b) in ((0, 0), (1, 1), (0, 1))
        m = imo.utterance_mask(1, 2, 5, 3, f, t)
        assert m[0].all() if b - a == 1 else not m[0].any()
        assert not m[1].any()
        widths.add(b - a)
    assert widths == {0, 1}


def test_utterance_shorter_than_the_context():
    """T_u = 2 < c = 7: every slot clamps into frames 0..1."""
    raw = imo.raw_frames(2, 2, 7)
    assert raw.tolist() == [[0, 0, 0, 0, 1, 1, 1], [0, 0, 0, 1, 1, 1, 1]]
    m = imo.utterance_mask(2, 3, 4, 7, [], [(1, 2)])
    assert np.array_equal(m[0].reshape(7, 4)[:, 0], raw[0] == 1) and not m[2].any()


def test_clamp_at_both_utterance_ends():
    raw = imo.raw_frames(10, 10, 5)
    assert raw[0].tolist() == [0, 0, 0, 1, 2] and raw[9].tolist() == [7, 8, 9, 9, 9]
    # masking frame 0 reaches rows 0..2 (their slots 0..2-row) and nothing else
    m = imo.utterance_mask(10, 10, 1, 5, [], [(0, 1)])
    assert m[:3].any(axis=1).all() and not m[3:].any()
    assert m[0].tolist() == [True, True, True, False, False]
    m = imo.utterance_mask(10, 10, 1, 5, [], [(9, 10)])
    assert m[7:].any(axis=1).all() and not m[:7].any()
    assert m[9].tolist() == [False, False, True, True, True]


@pytest.mark.parametrize("Tw,p", [(5, 0.0), (0, 1.0), (5, 0.05)])
def test_no_time_mask_when_W_is_zero(Tw, p):
    """W = min(T, floor(p T_u)) = 0 (p = 0, T = 0, or p T_u < 1 at T_u = 10): every time mask is empty."""
    for step in range(30):
        _, t = imo.bands(7, step, 3, 8, 10, 0, 0, 4, Tw, p)
        assert all(b == a for a, b in t)


def test_time_limit_is_floor_in_float64():
    assert imo.time_limit(10, 100, 0.7) == 7          # float32(0.7) * 10 would floor to 6
    assert imo.time_limit(100, 5, 1.0) == 5 and imo.time_limit(3, 100, 1.0) == 3


def test_no_frequency_mask_at_F_zero_and_whole_bands_at_F_nu():
    for step in range(30):
        f, _ = imo.bands(7, step, 3, 8, 10, 4, 0, 0, 0, 1.0)
        assert all(b == a for a, b in f)
    seen = set()
    for step in range(3000):
        f, _ = imo.bands(7, step, 3, 8, 10, 1, 8, 0, 0, 1.0)
        a, b = f[0]
        assert 0 <= a <= b <= 8
        seen.add(b - a)
    assert seen == set(range(9))                      # F = nu reaches the whole row


def test_without_splicing():
    """c = 1: slot 0 of row t' is frame t'."""
    assert imo.raw_frames(6, 6, 1)[:, 0].tolist() == list(range(6))
    m = imo.utterance_mask(6, 6, 4, 1, [(1, 3)], [(2, 4)])
    assert m[2:4].all() and m[[0, 1, 4, 5]][:, 1:3].all() and not m[[0, 1, 4, 5]][:, [0, 3]].any()


def test_counter_words_and_seed_halves_change_the_draws():
    base = imo.draws(5, 3, 7, 4)
    for other in (imo.draws(5, 4, 7, 4), imo.draws(5, 3, 8, 4), imo.draws(5 + 2 ** 32, 3, 7, 4)):
        assert not np.array_equal(base, other)
    assert np.array_equal(base, imo.draws(5, 3 + 2 ** 32, 7 + 2 ** 32, 4))     # step and g enter mod 2^32
    assert np.array_equal(base[:2], imo.draws(5, 3, 7, 2))                    # mask k's draw does not depend on the count


# ------------------------------------------------------------------------------------------------------- laws
def test_widths_and_starts_follow_their_uniform_laws():
    """w ~ U{0..F}; given w, f0 ~ U{0..nu - w}; chi-square over 20000 draws (utterances g of one step)."""
    nu, F, n = 41, 15, 20000
    ws, starts = [], []
    for g in range(n):
        (a, b), = imo.bands(9, 4, g, nu, 100, 1, F, 0, 0, 1.0)[0]
        ws.append(b - a)
        starts.append((a, b - a))
    counts = np.bincount(ws, minlength=F + 1)
    assert stats.chisquare(counts).pvalue > 1e-3, counts
    a8 = [a for a, w in starts if w == 8]
    assert stats.chisquare(np.bincount(a8, minlength=nu - 8 + 1)).pvalue > 1e-3
    # time masks: W = min(T, floor(p T_u)) = 20 at T_u = 100, p = 0.2; start uniform on 0..T_u - w
    tw, ta = [], []
    for g in range(n):
        (a, b), = imo.bands(9, 4, g, nu, 100, 0, 0, 1, 70, 0.2)[1]
        tw.append(b - a)
        if b - a == 20:
            ta.append(a)
    assert max(tw) == 20 and stats.chisquare(np.bincount(tw, minlength=21)).pvalue > 1e-3
    assert stats.chisquare(np.bincount(ta, minlength=81)).pvalue > 1e-3


# ------------------------------------------------------------------------------------------------------- C ABI
def _cfg(**kw):
    import _ctcb
    cfg = _ctcb.BrnnConfig(41 * 15, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def test_config_refusals_and_workspace_growth():
    from _ctcb import lib
    off = _cfg()
    assert off.maskFeatDim == 0          # an initialiser without the member keeps its meaning
    base = lib.ctcb_brnn_workspace_bytes(ctypes.byref(off))
    fwd = lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(off), None)
    err = lib.ctcb_brnn_error_flag_offset(ctypes.byref(off))
    assert base > 0
    for D, nu, why in ((615, -1, b"negative"), (615, 2, b"does not divide"), (615, 41 * 15 // 2, b"does not divide"),
                       (41 * 14, 41, b"odd"), (41 * 14, 41 * 7, b"odd"), (8, 1, b"odd")):
        cfg = _cfg(inputDim=D, maskFeatDim=nu)
        assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) == 0, nu
        h = ctypes.c_void_p()
        assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1, nu
        assert b"maskFeatDim" in lib.ctcb_last_error() and why in lib.ctcb_last_error(), lib.ctcb_last_error()
    copy = 60 * 8 * 41 * 15 * 4
    for nu in (41, 41 * 15, 1, 5, 123):
        cfg = _cfg(maskFeatDim=nu)
        got = lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg))
        assert got == base + (copy + 255) // 256 * 256, nu           # exactly the copy, rounded up to 256 bytes
        assert lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), None) == fwd
        assert lib.ctcb_brnn_error_flag_offset(ctypes.byref(cfg)) == err
        assert lib.ctcb_brnn_param_count(ctypes.byref(cfg)) == lib.ctcb_brnn_param_count(ctypes.byref(off))
    # a copy that is not a multiple of 256 bytes: inputDim 21 = 7 x 3, maxT 5, maxB 3
    cfg0 = _cfg(inputDim=21, maxT=5, maxB=3)
    cfg1 = _cfg(inputDim=21, maxT=5, maxB=3, maskFeatDim=7)
    assert (lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg1)) - lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg0))
            == 256 * ((5 * 3 * 21 * 4 + 255) // 256))
    # a layout too wide for the pass's bit sets
    wide = _cfg(inputDim=401001, maxT=2, maxB=1, maskFeatDim=1)
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(wide)) == 0
    assert lib.ctcb_brnn_create(ctypes.byref(wide), ctypes.byref(h)) == -1 and b"bit sets" in lib.ctcb_last_error()
    ok = _cfg(inputDim=300001, maxT=2, maxB=1, maskFeatDim=1)
    assert lib.ctcb_brnn_workspace_bytes(ctypes.byref(ok)) > 0


def test_set_input_masks_argument_contract():
    from _ctcb import lib
    step = ctypes.c_int64(0)     # the setter only stores the pointer: a host address does for the contract
    sp = ctypes.addressof(step)
    h, h0 = ctypes.c_void_p(), ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg(maskFeatDim=41)), ctypes.byref(h)) == 0
    assert lib.ctcb_brnn_create(ctypes.byref(_cfg()), ctypes.byref(h0)) == 0
    try:
        set_ = lib.ctcb_brnn_set_input_masks
        assert set_(h, 2, 15, 2, 70, 0.2, 33, sp) == 0
        assert set_(h, 64, 41, 64, 0, 0.0, 2 ** 64 - 1, sp) == 0
        assert set_(h, 0, 0, 0, 0, 1.0, 0, None) == 0                  # counts 0: off, no counter needed
        for bad in ((-1, 0, 0, 0, 1.0), (65, 0, 0, 0, 1.0), (0, 0, 65, 0, 1.0), (0, 0, -1, 0, 1.0), (1, 42, 0, 0, 1.0),
                    (1, -1, 0, 0, 1.0), (0, 0, 1, -1, 1.0), (0, 0, 1, 5, -0.1), (0, 0, 1, 5, 1.5),
                    (0, 0, 1, 5, float("nan")), (0, 0, 0, 0, 2.0)):
            assert set_(h, *bad, 1, sp) == -1, bad
            assert b"ctcb_brnn_set_input_masks" in lib.ctcb_last_error()
        assert set_(h, 1, 4, 0, 0, 1.0, 1, None) == -1 and b"step counter" in lib.ctcb_last_error()
        assert set_(h0, 1, 0, 0, 0, 1.0, 1, sp) == -1 and b"maskFeatDim" in lib.ctcb_last_error()
        assert set_(h0, 0, 4, 0, 3, 0.5, 1, None) == 0               # no layout, no masks: nothing to refuse
        assert set_(None, 0, 0, 0, 0, 1.0, 1, sp) == -1
    finally:
        lib.ctcb_brnn_destroy(h)
        lib.ctcb_brnn_destroy(h0)


def test_standalone_pass_refusals_launch_nothing():
    from _ctcb import lib
    step = ctypes.c_int64(0)
    sp, x = ctypes.addressof(step), ctypes.c_void_p(16)
    n0 = lib.ctcb_launch_count()
    f = lib.ctcb_input_mask_f32
    for args in ((x, x, 2, 3, 30, 7, 1, 1, 0, 0, 1.0, 1, sp, 0, 1, x),      # 7 does not divide 30
                 (x, x, 2, 3, 30, 15, 1, 1, 0, 0, 1.0, 1, sp, 0, 1, x),     # c = 2 is even
                 (x, x, 2, 3, 30, 10, 65, 1, 0, 0, 1.0, 1, sp, 0, 1, x),    # more than 64 masks
                 (x, x, 2, 3, 30, 10, 1, 11, 0, 0, 1.0, 1, sp, 0, 1, x),    # F > nu
                 (x, x, 2, 3, 30, 10, 1, 1, 0, 0, 1.0, 1, None, 0, 1, x),   # no counter
                 (x, x, 2, 3, 30, 10, 1, 1, 0, 0, 1.0, 1, sp, -1, 1, x),    # first < 0
                 (x, x, 2, 3, 30, 10, 1, 1, 0, 0, 1.0, 1, sp, 0, 0, x),     # stride < 1
                 (x, x, 0, 3, 30, 10, 1, 1, 0, 0, 1.0, 1, sp, 0, 1, x),     # B = 0
                 (x, None, 2, 3, 30, 10, 1, 1, 0, 0, 1.0, 1, sp, 0, 1, x)):
        assert f(*args, None) == -1, args
        assert b"ctcb_input_mask_f32" in lib.ctcb_last_error()
    assert lib.ctcb_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_mask_flags_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    d = runNNet._parse([])
    assert (d.freqMasks, d.freqMaskWidth, d.timeMasks, d.timeMaskWidth, d.timeMaskRatio, d.featDim) == (0, 0, 0, 0, 1.0,
                                                                                                         None)
    argv = ["--freqMasks", "2", "--freqMaskWidth", "15", "--timeMasks", "2", "--timeMaskWidth", "70",
            "--timeMaskRatio", "0.2", "--featDim", "41"]
    cfg = runNNet.run_config(runNNet._parse(argv))
    want = dict(freqMasks=2, freqMaskWidth=15, timeMasks=2, timeMaskWidth=70, timeMaskRatio=0.2, featDim=41)
    assert {k: cfg[k] for k in want} == want
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    resumed = runNNet.run_config(runNNet._parse(["--cfg_file", f]))
    assert {k: resumed[k] for k in want} == want
    old = {k: v for k, v in cfg.items() if k not in want}
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    got = runNNet.run_config(runNNet._parse(["--cfg_file", f2]))
    assert (got["freqMasks"], got["timeMasks"], got["featDim"]) == (0, 0, None)
    assert runNNet.trained_config(f2).timeMasks == 0
