"""CPU tests of the log-domain blank-forced CTC oracle (oracle.ctc_oracle.ctc_loss_blankforce_log), of where the
reference's arithmetic leaves float64's range, and of the best-path decoders' argmax.

The reference (ctc_fast_blankforce.pyx, restated bit-exact as oracle.ctc_oracle.ctc_loss_blankforce) normalises alpha
and beta per frame and multiplies them for the occupancies.  On long utterances with unaligned outputs:
  * the product underflows while the loss stays right: rows of the gradient are left at p;
  * the normalised trellis loses mass: the loss is wrong too.
The blank-forced cost sums the mass of ALL states at the last frame while beta starts from the last state only, so the
reference's discarded llBackward is not a check of its llForward; the second failure is recognised by the loss's
distance from the log-domain one instead.  Where the scaled oracle is in range the two oracles agree to rounding."""
import numpy as np
import pytest

import recipes
from oracle import ctc_oracle

GRAD_TOL, NLL_TOL = 1e-6, 1e-8


def _agree(p, seq):
    nll, g, skip = ctc_oracle.ctc_loss_blankforce(p, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_blankforce_log(p, seq)
    assert skip == lskip, (skip, lskip)
    if skip:                          # the reference's gradient is what it had accumulated when it stopped
        assert not lg.any()
        return True
    assert np.abs(g - lg).max() <= GRAD_TOL, np.abs(g - lg).max()
    if np.isinf(nll):
        assert lnll == nll
    else:
        assert abs(nll - lnll) <= NLL_TOL * max(1.0, abs(nll)), (nll, lnll)
    return False


@pytest.mark.parametrize("name", recipes.ALL_BF)
def test_log_oracle_equals_scaled_on_golden_cases(name):
    probs, seq = recipes.bf_case(name)
    assert not _agree(np.asfortranarray(probs.astype(np.float64)), seq)


def test_log_oracle_equals_scaled_on_random_cases():
    skips = [_agree(p, seq) for p, seq in recipes.random_bf_cases()]
    assert len(skips) == 200


def bf_edges(K=12, seed=5):
    """(name, probabilities float32 T x K, seq, skip) of one utterance per edge of the blank-forced trellis; the zero
    probabilities are exact."""
    rng = np.random.RandomState(seed)
    rows = []

    def add(name, T, seq, skip=False, edit=None):
        p = recipes.softmax64(rng.randn(T, K) * 1.5)
        if edit is not None:
            edit(p)
        rows.append((name, p.astype(np.float32), np.asarray(seq, np.int32), skip))
    lab = lambda n: np.insert(1 + rng.randint(K - 1, size=n), np.arange(n + 1), 0)[:2 * n + 1].astype(np.int32)

    def far_row0(p):                                                # p[0, t] far from p[seq[0], t]
        p[:, 0] *= 1e-5
        p /= p.sum(axis=1, keepdims=True)

    def zero(t, k):
        def f(p):
            p[t, k] = 0.0
            p /= p.sum(axis=1, keepdims=True)
        return f

    def zero_frame(t):
        def f(p):
            p[t] = 0.0
        return f

    def zero_col(k):
        def f(p):
            p[:, k] = 0.0
            p /= p.sum(axis=1, keepdims=True)
        return f
    add("T1_L1", 1, [0]); add("T1_L1_label", 1, [4]); add("T1_L5", 1, lab(2)); add("T2_L3", 2, lab(1))
    add("T2_L1", 2, [7]); add("T_eq_L", 9, lab(4)); add("T_lt_L_overlap", 7, lab(4))
    add("T_lt_L_apart", 4, lab(5)); add("row0_quirk", 30, [5, 0, 3, 0, 7, 0], edit=far_row0)
    add("row0_quirk_L1", 12, [6], edit=far_row0)
    add("zero_p_L1_last_frame", 6, [4], skip=True, edit=zero(5, 4))           # alpha uses row 0, the gradient row 4
    add("zero_p_T1_L1", 1, [4], skip=True, edit=zero(0, 4))
    add("zero_beta_frame", 6, [4], skip=True, edit=zero(2, 4))                 # beta's normaliser 0 from frame 2 down
    add("zero_frame", 10, lab(2), skip=True, edit=zero_frame(4))
    add("zero_on_only_path", 6, [0], skip=True, edit=zero(3, 0))
    add("zero_label_elsewhere", 25, lab(5), edit=zero_col(K - 1))
    add("zero_first_state_frame0", 8, [3, 0, 5], edit=zero(0, 3))               # nll = inf, gradient computed
    return rows


EDGES = bf_edges()


@pytest.mark.parametrize("case", EDGES, ids=[e[0] for e in EDGES])
def test_log_oracle_equals_scaled_on_trellis_edges(case):
    name, p, seq, skip = case
    p64 = np.asfortranarray(p.T.astype(np.float64))
    assert _agree(p64, seq) == skip
    lnll, lg, _ = ctc_oracle.ctc_loss_blankforce_log(p64, seq)
    if name == "T_lt_L_apart":                                     # alpha and beta never meet: rows stay p, loss finite
        assert np.array_equal(lg, p64) and np.isfinite(lnll)
    if name == "zero_first_state_frame0":
        assert lnll == np.inf and not np.array_equal(lg, p64)


def test_empty_utterances_skip():
    p = np.asfortranarray(np.full((5, 3), 0.2))
    assert ctc_oracle.ctc_loss_blankforce_log(p, np.zeros(0, np.int32))[2]
    assert ctc_oracle.ctc_loss_blankforce_log(np.asfortranarray(np.zeros((5, 0))), np.zeros(1, np.int32))[2]


def _utt(T, nlab, scale, seed, K=40):
    x, seq = recipes.bf_utt(T, K, nlab, scale, seed)
    return np.asfortranarray(recipes.softmax64(x).T), seq


def _log_forward_nll(p, seq):
    """An independent log-domain forward pass (numpy, vectorised over states)."""
    with np.errstate(divide="ignore"):
        lp = np.log(p)
    row = seq.copy()
    row[0] = 0                                                    # the alpha pass's row-0 quirk
    a = np.full(len(seq), -np.inf)
    a[0] = 0.0
    for t in range(1, p.shape[1]):
        a = np.logaddexp(a, np.concatenate([[-np.inf], a[:-1]])) + lp[row, t]
    return -(lp[seq[0], 0] + np.logaddexp.reduce(a))


# Measured with the two oracles on recipes.bf_utt (K = 40, float64 softmax of the float32 logits): T, labels, scale,
# seed, then the frames on which the scaled gradient is off by more than 1e-6 and the rows it left at exactly p.
IN_RANGE = [(1500, 150, 2.0, 1), (1500, 150, 3.0, 1)]
UNDERFLOW = [(1500, 150, 3.0, 3, 28, 0), (3000, 300, 2.0, 1, 847, 805), (3000, 300, 3.0, 3, 1454, 1429)]
# ... and the distance of the scaled loss from the log-domain one, in nats
LOST_MASS = [(5000, 300, 2.0, 1, 32.118), (5000, 300, 3.0, 3, 264.514)]


@pytest.mark.parametrize("T,nlab,scale,seed", IN_RANGE)
def test_in_range_long_utterances_agree(T, nlab, scale, seed):
    p, seq = _utt(T, nlab, scale, seed)
    assert not _agree(p, seq)


@pytest.mark.parametrize("T,nlab,scale,seed,bad,at_p", UNDERFLOW)
def test_product_underflow_leaves_rows_at_p(T, nlab, scale, seed, bad, at_p):
    """The scaled loss is right, but on the bad frames its gradient is p (or computed from a subnormal absum)."""
    p, seq = _utt(T, nlab, scale, seed)
    nll, g, skip = ctc_oracle.ctc_loss_blankforce(p, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_blankforce_log(p, seq)
    assert not skip and not lskip
    assert abs(nll - lnll) <= NLL_TOL * lnll, (nll, lnll)
    assert abs(lnll - _log_forward_nll(p, seq)) <= 1e-10 * lnll
    off = np.abs(g - lg).max(axis=0) > GRAD_TOL
    rows_p = (g == p).all(axis=0)
    assert off.sum() == bad and rows_p.sum() == at_p and not (rows_p & ~off).any()
    assert np.abs(lg.sum(axis=0)).max() <= 1e-9                   # every log-domain row of softmax outputs sums to 0
    assert np.abs(g[:, ~off] - lg[:, ~off]).max() <= GRAD_TOL


@pytest.mark.parametrize("T,nlab,scale,seed,dnll", LOST_MASS)
def test_lost_trellis_mass_gives_a_wrong_loss(T, nlab, scale, seed, dnll):
    """5000 frames, 601 states: the scaled trellis loses mass, its loss is off by tens to hundreds of nats and most rows
    are p.  The log-domain loss agrees with an independent forward pass and its rows sum to 0."""
    p, seq = _utt(T, nlab, scale, seed)
    nll, g, skip = ctc_oracle.ctc_loss_blankforce(p, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_blankforce_log(p, seq)
    assert not skip and not lskip
    assert abs(abs(nll - lnll) - dnll) <= 1e-3, (nll, lnll)
    assert abs(lnll - _log_forward_nll(p, seq)) <= 1e-10 * lnll
    assert np.abs(lg.sum(axis=0)).max() <= 1e-9
    assert (np.abs(g - lg).max(axis=0) > GRAD_TOL).sum() >= 4000


# ---- best path: np.argmax per frame, then the collapse of ctc_fast.pyx:154-187 / ctc_fast_blankforce.pyx:115-142
def np_best_path(probs, blank=0, drop=True):
    """probs K x T.  np.argmax picks the first NaN, else the first maximum."""
    hyp, align, prev = [], [], -1
    for t in range(probs.shape[1]):
        b = int(np.argmax(probs[:, t]))
        if b == blank or (drop and b in (1, 2, 8)):
            prev = b
            continue
        if t != 0 and b == prev:
            if hyp:
                align[-1] = t
            continue
        hyp.append(b)
        align.append(t)
        prev = b
    return hyp, align


def awkward_rows(K, T, seed):
    """K x T float32 rows with NaN (at 0, inside, everywhere), +-inf, all -inf, ties across lanes and runs of repeats."""
    rng = np.random.RandomState(seed)
    p = rng.randint(0, 4, size=(K, T)).astype(np.float32)          # many ties
    kinds = rng.randint(0, 8, size=T)
    for t, kind in enumerate(kinds):
        if kind == 1:
            p[0, t] = np.nan
        elif kind == 2:
            p[rng.randint(K), t] = np.nan
            p[rng.randint(K), t] = np.nan
        elif kind == 3:
            p[:, t] = np.nan
        elif kind == 4:
            p[:, t] = -np.inf
        elif kind == 5:
            p[rng.randint(K), t] = np.inf
            p[rng.randint(K), t] = np.inf
        elif kind == 6 and t > 0:
            p[:, t] = p[:, t - 1]                                  # a repeat
    return p


@pytest.mark.parametrize("K", [2, 5, 31, 33, 70])
def test_decoders_follow_np_argmax(K):
    with np.errstate(invalid="ignore"):
        for seed in range(4):
            p = awkward_rows(K, 200, seed + 17 * K).astype(np.float64)
            for blank in (0, K // 2, K - 1):
                hyp, align = ctc_oracle.decode_best_path(np.asfortranarray(p), blank)
                assert (hyp, align) == np_best_path(p, blank)
                assert ctc_oracle.decode_best_path_blankforce(np.asfortranarray(p), blank) == \
                    np_best_path(p, blank, drop=False)[0]
