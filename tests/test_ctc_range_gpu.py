"""GPU test of the CTC kernel (ctcb_ctc_loss_grad_f32) on long utterances, against the log-domain float64 oracle
(oracle.ctc_oracle.ctc_loss_log), on every kernel organisation.

The scaled float64 oracle (the reference's arithmetic) is not the truth here.  On long utterances with unaligned outputs
its per-frame product of normalised alpha and beta underflows (grad rows left at p: tests/test_ctc_range_cpu.py), and
further out its trellis loses mass (wrong loss; its llForward and llBackward disagree).  Every case below is classified
by the two CPU oracles, and each out-of-range case asserts that it is out of range, so none can pass on an in-range input
by accident:
  in        the oracles agree (gradient to 1e-6, loss to 1e-8 relative);
  underflow the gradients differ but the scaled loss is right (forward and backward agree to 1e-6 nats);
  lost      the scaled trellis lost mass (forward and backward differ by more than 1e-3 nats).
Per utterance: skip = 1 with a zero gradient, or skip = 0 with max |g - g_log| and the NLL error inside the
organisation's BOUNDS (test_ctc_plans_gpu.py); every "in" and every "underflow" utterance has skip = 0 (and so a correct
gradient); with logits input every gradient row of a computed utterance sums to 0 within ROW_SUM_BOUND.
Each case prints one JSON line: plan, errors, skips per class, and a digest of the kernel's outputs."""
import functools
import hashlib
import json
import time

import numpy as np
import pytest

import recipes
from oracle import ctc_oracle
from recipes import Batch, knobs  # noqa: F401  (knobs: fixture)
from test_ctc_plans_gpu import BOUNDS, H100_SMS, SENTINEL, _run, force  # noqa: F401  (force: fixture)

pytestmark = pytest.mark.gpu
ROW_SUM_BOUND = 1e-4      # |sum_k g[t, k]|, logits input: e/Z sums to 1 in float32, the 2^30 fixed-point occupancies to 1

# (T, K, |l|, logit scale, seed, class) -- utterances of recipes.ctc_batch(1, T, K, |l|, seed, ragged=False, scale=...)
IN = [(200, 62, 30, 2.0, 1, "in"), (1500, 35, 150, 2.0, 1, "in"), (1500, 35, 150, 2.0, 5, "in")]
UNDER = [(1500, 35, 150, 3.0, 3, "underflow"), (1500, 35, 150, 3.0, 6, "underflow"), (2000, 35, 200, 2.0, 1, "underflow"),
         (3000, 35, 300, 2.0, 1, "underflow")]
LOST = [(5000, 35, 300, 2.0, 11, "lost"), (5000, 35, 300, 0.1, 1, "lost")]
# |l| <= 127 (the checkpoint kernel's P <= 4) and |l| <= 63 (P <= 2, the warp kernel's 8-frame tiles), chosen by the oracles
SMALL = [(1500, 35, 100, 2.0, 1, "in"), (1500, 35, 127, 3.0, 1, "underflow"), (3000, 35, 63, 2.0, 1, "underflow"),
         (3000, 35, 127, 3.0, 1, "lost"), (3000, 35, 63, 3.0, 1, "lost")]
P2 = [(1500, 35, 60, 2.0, 1, "in"), (3000, 35, 63, 2.0, 1, "underflow"), (3000, 35, 63, 3.0, 1, "lost")]


@functools.lru_cache(maxsize=None)
def _utt(T, K, L, scale, seed, is_prob):
    """(x float32 T x K, labels, p float64 T x K) of one utterance; probability input is the float32 softmax."""
    b = recipes.ctc_batch(1, T, K, L, seed, ragged=False, scale=scale)
    x = b.x[0]
    if is_prob:
        x = recipes.softmax64(x).astype(np.float32)
    p = x.astype(np.float64) if is_prob else recipes.softmax64(x)
    return x, b.seqs[0], p


@functools.lru_cache(maxsize=None)
def _oracles(case, is_prob):
    """Log-domain result and the class the two CPU oracles give the utterance."""
    T, K, L, scale, seed, _ = case
    _, seq, p = _utt(T, K, L, scale, seed, is_prob)
    pf = np.asfortranarray(p.T)
    nll, g, skip, llb = ctc_oracle.ctc_loss_fb(pf, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_log(pf, seq)
    assert not skip and not lskip
    gdiff = float(np.abs(g - lg).max())
    fb = abs(-nll - llb)
    if gdiff <= 1e-6 and abs(nll - lnll) <= 1e-8 * lnll:
        cls = "in"
    elif fb <= 1e-6 and abs(nll - lnll) <= 1e-6 * lnll:
        cls = "underflow"
    elif fb > 1e-3:
        cls = "lost"
    else:
        cls = "between"
    return lnll, lg.T.copy(), cls


def _batch(cases, is_prob, copies=1, layout="bt"):
    xs = [_utt(c[0], c[1], c[2], c[3], c[4], is_prob) for c in cases] * copies
    Tmax, K = max(x.shape[0] for x, _, _ in xs), cases[0][1]
    x = np.zeros((len(xs), Tmax, K), np.float32)
    for u, (xu, _, _) in enumerate(xs):
        x[u, :xu.shape[0]] = xu
    return Batch(x, [xu.shape[0] for xu, _, _ in xs], [s for _, s, _ in xs], is_prob=is_prob, layout=layout)


def _check(torch, force, name, cases, forced, expect, is_prob, copies=1, layout="bt"):
    t0 = time.time()
    for c in cases:                                   # every case is what it claims to be
        assert _oracles(c, is_prob)[2] == c[5], (c, _oracles(c, is_prob)[2])
    b = _batch(cases, is_prob, copies, layout)
    force(forced)
    plan, nll, g, skip, gaps = _run(torch, b, plan_expect=expect, what=name)
    assert (gaps == SENTINEL).all(), "the kernel wrote outside the gradient's elements"
    gb, nb = BOUNDS[plan["kernel"]]
    gerr = nerr = rowsum = 0.0
    n = {}
    for u in range(b.B):
        c = cases[u % len(cases)]
        T = b.lens[u]
        lnll, lg, cls = _oracles(c, is_prob)
        key = "%s-%s" % (cls, "skip" if skip[u] else "ok")
        n[key] = n.get(key, 0) + 1
        assert skip[u] in (0, 1)
        assert not g[u, T:].any()
        if skip[u]:
            assert not g[u].any(), "skipped utterance %d has a gradient" % u
            assert cls == "lost", ("utterance %d (%s, %s) skipped" % (u, c, cls), nll[u], lnll)
            continue
        ge = float(np.abs(g[u, :T] - lg).max())
        ne = abs(nll[u] - lnll) / lnll
        assert ge <= gb and ne <= nb, (u, c, cls, ge, ne, gb, nb)
        gerr, nerr = max(gerr, ge), max(nerr, ne)
        if not is_prob:
            rowsum = max(rowsum, float(np.abs(g[u, :T].sum(axis=1)).max()))
    digest = hashlib.sha256(nll.astype(np.float32).tobytes() + g.astype(np.float32).tobytes()
                            + skip.astype(np.int32).tobytes()).hexdigest()[:16]
    print(json.dumps(dict(ctc=name, plan=plan, forced=forced, is_prob=is_prob, B=b.B, Tmax=b.Tmax, grad_err=gerr,
                          nll_err=nerr, grad_bound=gb, nll_bound=nb, row_sum=rowsum, utterances=n, digest=digest,
                          seconds=round(time.time() - t0, 2))))
    assert rowsum <= ROW_SUM_BOUND, rowsum


ORGS = [("par", "auto", dict(kernel="par", P=16)), ("pair", "pair", dict(kernel="pair", P=16)),
        ("warp16", "warp", dict(kernel="warp", th=16, nbuf=2, P=16))]


@pytest.mark.parametrize("is_prob", [False, True], ids=["logit", "prob"])
@pytest.mark.parametrize("case", IN + UNDER + LOST, ids=lambda c: "T%d-L%d-s%g-seed%d-%s" % (c[0], c[2], c[3], c[4], c[5]))
@pytest.mark.parametrize("org,forced,expect", ORGS, ids=[o[0] for o in ORGS])
def test_long_utterance(org, forced, expect, case, is_prob, cuda, force):
    """One utterance per launch at P = 16 (up to 511 labels); par is the default plan for a single utterance."""
    exp = dict(expect, P=16 if case[2] > 255 else 8 if case[2] > 127 else 4 if case[2] > 63 else 2 if case[2] > 31 else 1)
    _check(cuda, force, "range-%s" % org, [case], forced, exp, is_prob)


@pytest.mark.parametrize("is_prob", [False, True], ids=["logit", "prob"])
@pytest.mark.parametrize("org,forced,expect", [("ckpt", "ckpt", dict(kernel="ckpt", P=4)),
                                               ("par", "par", dict(kernel="par", P=4)),
                                               ("warp16", "warp", dict(kernel="warp", th=16, nbuf=2, P=4))],
                         ids=["ckpt", "par", "warp16"])
def test_checkpoint_reachable(org, forced, expect, is_prob, cuda, force):
    """|l| <= 127: every class in one batch, on the checkpoint kernel and, for the same inputs, par and warp."""
    _check(cuda, force, "range-small-%s" % org, SMALL, forced, expect, is_prob)


def test_warp_8_frame_tiles(cuda, force):
    """The warp kernel's 8-frame tiles with one buffer need a batch of 16 x SMs utterances and |l| <= 63 (P <= 2):
    the three classes, repeated."""
    copies = (16 * H100_SMS + len(P2) - 1) // len(P2)
    _check(cuda, force, "range-warp8", P2, "warp", dict(kernel="warp", th=8, nbuf=1, P=2), False, copies=copies)


@pytest.mark.parametrize("org,forced", [("par", "auto"), ("pair", "pair"), ("ckpt", "ckpt"), ("warp", "warp")])
def test_ragged_time_major_mixed(org, forced, cuda, force):
    """A ragged time-major batch (the BRNN's layout) mixing in-range, underflowing and mass-losing utterances of
    different lengths."""
    cases = [SMALL[0], SMALL[2], SMALL[3], SMALL[1], SMALL[4]]
    _check(cuda, force, "range-ragged-%s" % org, cases, forced, dict(kernel=org), False, layout="tb")
