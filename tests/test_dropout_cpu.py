"""CPU tests of inverted dropout on the ReLU hidden layers (ctcb_brnn_set_dropout): the NumPy mask of
tests/net_oracle.py against the published Philox4x32-10 answers and for its statistics, the float64 net with dropout
back-propagating through given activations as through its own, the minibatch index g of every utterance however a step
is sharded and cut, the setters' argument contract through the C ABI (host-only calls, no device), and the runNNet flag.
No compute call is made on a device here."""
import ctypes
import math

import numpy as np
import pytest

import parallel
from net_oracle import Net, draws, keep_mask, philox4x32_10, threshold_scale


# ---------------------------------------------------------------------------------------------------------- Philox
def test_philox_known_answers():
    """The known-answer vectors of Philox4x32-10 (Random123, kat_vectors): zero, all-ones and pi-digit counters/keys."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]
        assert tuple(int(x) for x in got) == want


def test_threshold_and_scale():
    assert threshold_scale(0.5) == (2 ** 31, np.float32(2.0))
    thr, s = threshold_scale(0.1)
    assert thr == math.floor(float(np.float32(0.1)) * 2 ** 32) and s == np.float32(1.0 / (1.0 - float(np.float32(0.1))))
    assert threshold_scale(0.0) == (0, np.float32(1.0))
    assert threshold_scale(np.nextafter(np.float32(1), np.float32(0)))[0] < 2 ** 32


@pytest.mark.parametrize("p", [0.05, 0.1, 0.5])
def test_keep_fraction_is_one_minus_p(p):
    """Over 2500 frames x 4096 units (1.02e7 draws) the kept fraction is within 6 sigma of 1 - p."""
    keep = keep_mask(p, 33, 7, 2, 5, 2500, 4096)
    n = keep.size
    assert n >= 10 ** 7
    frac = keep.mean()
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(frac - (1 - p)) < 6 * sigma, (frac, 1 - p, sigma)


def _corr(a, b):
    a, b = a.astype(np.float64).ravel(), b.astype(np.float64).ravel()
    return float(np.corrcoef(a, b)[0, 1])


def test_masks_of_different_steps_layers_utterances_and_seeds_are_uncorrelated():
    """Change one argument at a time (step, layer, utterance, seed's low and high word, frame offset): the two masks
    differ and their correlation is within 6 / sqrt(n) of 0."""
    p, T, H = 0.3, 400, 1000
    base = dict(seed=33, step=4, layer=2, g=9)
    ref = keep_mask(p, T=T, H=H, **base)
    bound = 6.0 / math.sqrt(T * H)
    for key, val in [("step", 5), ("layer", 3), ("g", 10), ("g", 9 + 2 ** 20), ("seed", 34), ("seed", 33 + 2 ** 32)]:
        other = keep_mask(p, T=T, H=H, **dict(base, **{key: val}))
        assert not np.array_equal(ref, other), key
        assert abs(_corr(ref, other)) < bound, (key, val, _corr(ref, other))
    # frames and units of one mask are not copies of each other either
    assert abs(_corr(ref[:-1], ref[1:])) < bound and abs(_corr(ref[:, :-1], ref[:, 1:])) < bound


def test_units_beyond_the_last_float4_are_drawn_like_the_rest():
    """H not a multiple of 4: the tail units are the first outputs of the last group's draw."""
    full = draws(1, 2, 3, 4, 6, 12)
    tail = draws(1, 2, 3, 4, 6, 10)
    assert np.array_equal(full[:, :10], tail)


# ------------------------------------------------------------------------------------------ minibatch index g
@pytest.mark.parametrize("n,world,cap", [(13, 1, 13), (13, 1, 4), (13, 2, 3), (17, 4, 2), (7, 3, 5), (2, 4, 1)])
def test_each_minibatch_utterance_gets_one_index_however_the_step_is_split(n, world, cap):
    """g = rank + world * (u0 + u): the round-robin shard of rank r (parallel.shard) cut into consecutive micro-batches
    (parallel.micro_batches) starting at shard position u0 gives utterance u the position of that utterance in the
    whole step, so every utterance gets exactly one index and the same one as in a single call."""
    step = ["utt%d" % i for i in range(n)]
    seen = {}
    for r in range(world):
        pieces = parallel.micro_batches(parallel.shard(step, r, world), cap)
        u0 = 0
        for piece in pieces:
            for u, key in enumerate(piece):
                g = r + world * (u0 + u)
                assert key not in seen
                seen[key] = g
            u0 += len(piece)
    assert seen == {key: i for i, key in enumerate(step)}


# ---------------------------------------------------------------------------------------- the float64 restatement
def test_back_propagation_through_given_activations_is_the_same():
    """costAndGradGiven on the net's own dropped activations = costAndGrad (the GPU tests feed it the device's)."""
    np.random.seed(2)
    nn = Net(7, 5, 12, 4, 9, temporalLayer=2, round_f32=False, dropout=0.5, dropoutSeed=1)
    nn.initParams()
    nn.dropoutStep, nn.utt = 2, 3
    data = np.random.RandomState(1).randn(7, 9)
    labels = np.array([1, 3, 2], dtype=np.int32)
    c1, g1, _ = nn.costAndGrad(data, labels)
    g1 = [[a.copy(), b.copy()] for a, b in g1]
    h, temporal, _ = nn.forward(data)
    c2, g2, _ = nn.costAndGradGiven(data, labels, h[1:], temporal)
    assert c1 == c2
    for (a, b), (x, y) in zip(g1, g2):
        assert np.array_equal(a, x) and np.array_equal(b, y)


# --------------------------------------------------------------------------------------------------- C ABI
def _handle():
    import _ctcb
    from _ctcb import lib
    cfg = _ctcb.BrnnConfig(13, 11, 64, 3, 2, 60, 8, 20, 0.0, 20.0, 0, 1)
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return lib, h


def test_set_dropout_argument_contract():
    lib, h = _handle()
    try:
        step = ctypes.c_int64(0)     # the setters only store the pointer: a host address does for the contract
        sp = ctypes.addressof(step)
        for p in (-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf")):
            assert lib.ctcb_brnn_set_dropout(h, p, 1, sp) == -1, p
            assert b"ctcb_brnn_set_dropout" in lib.ctcb_last_error()
        assert lib.ctcb_brnn_set_dropout(h, 0.1, 1, None) == -1 and b"step counter" in lib.ctcb_last_error()
        assert lib.ctcb_brnn_set_dropout(h, 0.0, 1, None) == 0          # p == 0 disables and needs no counter
        assert lib.ctcb_brnn_set_dropout(h, 0.1, 2 ** 64 - 1, sp) == 0
        assert lib.ctcb_brnn_set_dropout(h, 0.999, 0, sp) == 0
        assert lib.ctcb_brnn_set_dropout(None, 0.1, 1, sp) == -1
        for first, stride in ((0, 0), (0, -1), (-1, 1), (3, -2)):
            assert lib.ctcb_brnn_set_dropout_utts(h, first, stride) == -1, (first, stride)
        assert lib.ctcb_brnn_set_dropout_utts(h, 3, 2) == 0
        assert lib.ctcb_brnn_set_dropout_utts(h, 2 ** 40, 2 ** 20) == 0
        assert lib.ctcb_brnn_set_dropout_utts(None, 0, 1) == -1
        n0 = lib.ctcb_launch_count()
        assert lib.ctcb_dropout_advance(None, None) == -1
        assert lib.ctcb_launch_count() == n0
    finally:
        lib.ctcb_brnn_destroy(h)


# ---------------------------------------------------------------------------------------------------- runNNet
def test_runnnet_dropout_flag_and_old_configs(tmp_path):
    import runNNet
    from run_utils import dump_config
    assert runNNet._parse([]).dropout == 0.0
    cfg = runNNet.run_config(runNNet._parse(["--dropout", "0.1"]))
    assert cfg["dropout"] == 0.1
    f = str(tmp_path / "cfg.json")
    dump_config(cfg, f)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f]))["dropout"] == 0.1      # resume keeps it
    old = dict(cfg)
    del old["dropout"]
    f2 = str(tmp_path / "old_cfg.json")
    dump_config(old, f2)
    assert runNNet.run_config(runNNet._parse(["--cfg_file", f2]))["dropout"] == 0.0     # a run from before the flag
    assert runNNet.trained_config(f2).dropout == 0.0
