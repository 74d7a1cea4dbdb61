"""CPU tests of the log-domain CTC oracle (oracle.ctc_oracle.ctc_loss_log) and of where the reference's arithmetic
leaves float64's range.

The reference (ctc_fast.pyx, restated bit-exact as oracle.ctc_oracle.ctc_loss) normalises alpha and beta per frame and
multiplies them to get the occupancies.  On long utterances with unaligned outputs two things go wrong:
  * the product underflows while the loss stays right: absum of a frame falls below 1e-308, the gradient row is left at
    p (or computed from a few bits), and its occupancies sum to 0 instead of 1;
  * the trellis itself loses mass: the loss is wrong too, and the llBackward the reference computes and discards
    disagrees with its llForward.
The log-domain oracle has neither problem.  Where the scaled oracle is in range the two agree to rounding."""
import numpy as np
import pytest

import recipes
from oracle import ctc_oracle

TOL = 1e-10


def _utt(T, K, L, scale, seed):
    """Float64 probabilities (K x T, F-order) and labels of one utterance of recipes.ctc_batch (logits input)."""
    b = recipes.ctc_batch(1, T, K, L, seed, ragged=False, scale=scale)
    return np.asfortranarray(recipes.softmax64(b.x[0]).T), b.seqs[0]


def _agree(p, seq, blank=0):
    nll, g, skip = ctc_oracle.ctc_loss(p, seq, blank)
    lnll, lg, lskip = ctc_oracle.ctc_loss_log(p, seq, blank)
    assert skip == lskip, (skip, lskip)
    if skip:
        assert not lg.any()
        return
    assert np.abs(g - lg).max() <= TOL, np.abs(g - lg).max()
    if np.isinf(nll):
        assert np.isinf(lnll) and lnll > 0
    else:
        assert abs(nll - lnll) <= TOL * max(1.0, abs(nll)), (nll, lnll)


@pytest.mark.parametrize("name", recipes.ALL_CTC)
def test_log_oracle_equals_scaled_on_golden_cases(name):
    probs, seq = recipes.ctc_case(name)
    _agree(np.asfortranarray(probs.astype(np.float64)), seq)


def test_log_oracle_equals_scaled_on_random_shapes():
    for p, seq in recipes.random_ctc_cases():
        _agree(p, seq)


@pytest.mark.parametrize("is_prob", [False, True])
def test_log_oracle_equals_scaled_on_trellis_edges(is_prob):
    K = 12
    rng = np.random.RandomState(4)
    skips = []
    for T, seq in recipes.ctc_trellis_edges(K):
        p = recipes.softmax64(rng.randn(T, K) * 1.5)
        if is_prob:
            p[:, 3] = 0.0                                    # exact zeros, label 3 impossible
            p /= p.sum(axis=1, keepdims=True)
        _agree(np.asfortranarray(p.T), seq)
        skips.append(ctc_oracle.ctc_loss_log(np.asfortranarray(p.T), seq)[2])
    if is_prob:                                              # every sequence that needs label 3 has no alignment
        assert skips == [3 in seq and 2 <= T and len(seq) <= T for T, seq in recipes.ctc_trellis_edges(K)]
    else:
        assert skips[5] and not any(skips[i] for i in (4, 6, 7, 8))


def test_log_oracle_blank_inside_sequence_and_not_zero():
    rng = np.random.RandomState(8)
    K, T = 9, 30
    p = np.asfortranarray(recipes.softmax64(rng.randn(T, K)).T)
    for blank, seq in ((4, [1, 4, 4, 2, 4]), (8, [1, 2, 2, 3]), (0, [5])):
        _agree(p, np.asarray(seq, np.int32), blank)


def _log_forward_nll(p, seq):
    """An independent log-domain forward pass (numpy, vectorised over states): -log P(l|x)."""
    L = 2 * len(seq) + 1
    lab = np.zeros(L, np.int64)
    lab[1::2] = seq
    skip = np.zeros(L, bool)
    skip[3::2] = np.asarray(seq[1:]) != np.asarray(seq[:-1])
    with np.errstate(divide="ignore"):
        lp = np.log(p)
    a = np.full(L, -np.inf)
    a[:2] = lp[lab[:2], 0]
    for t in range(1, p.shape[1]):
        a1 = np.concatenate([[-np.inf], a[:-1]])
        a2 = np.where(skip, np.concatenate([[-np.inf, -np.inf], a[:-2]]), -np.inf)
        a = np.logaddexp(np.logaddexp(a, a1), a2) + lp[lab, t]
    return -np.logaddexp(a[-1], a[-2])


# Rows measured with the two oracles (logits ~ N(0, scale^2), float64 softmax): T, K, |l|, scale, seed, frames on which
# the scaled oracle's gradient is off by more than 1e-6.
IN_RANGE = [(200, 62, 30, 2.0, 1), (800, 32, 100, 3.0, 2), (1500, 35, 150, 2.0, 1), (1500, 35, 150, 2.0, 5)]
# The last column: of those, the frames whose absum underflowed to exactly 0 (the others kept a few bits of it).
UNDERFLOW = [(1500, 35, 150, 3.0, 3, 475, 445), (1500, 35, 150, 3.0, 6, 352, 202), (2000, 35, 200, 2.0, 1, 424, 277),
             (3000, 35, 300, 2.0, 1, 1695, 1672)]
LOST_MASS = [(5000, 35, 300, 2.0, 11), (5000, 35, 300, 0.1, 1)]


@pytest.mark.parametrize("T,K,L,scale,seed", IN_RANGE)
def test_in_range_long_utterances_agree(T, K, L, scale, seed):
    p, seq = _utt(T, K, L, scale, seed)
    _agree(p, seq)
    nll, _, _, llb = ctc_oracle.ctc_loss_fb(p, seq)
    assert abs(-nll - llb) <= 1e-9


@pytest.mark.parametrize("T,K,L,scale,seed,bad,at_p", UNDERFLOW)
def test_product_underflow_leaves_rows_at_p(T, K, L, scale, seed, bad, at_p):
    """The loss is right (forward and backward agree, and agree with the log domain), but on the bad frames the scaled
    oracle's gradient is wrong: most rows are p and sum to sum_k p = 1, where a gradient row of softmax outputs sums to
    0; the rest come from the few bits of a subnormal absum."""
    p, seq = _utt(T, K, L, scale, seed)
    nll, g, skip, llb = ctc_oracle.ctc_loss_fb(p, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_log(p, seq)
    assert not skip and not lskip
    assert abs(-nll - llb) <= 1e-7 and abs(nll - lnll) <= 1e-7, (nll, llb, lnll)
    assert abs(lnll - _log_forward_nll(p, seq)) <= 1e-9 * lnll
    off = np.abs(g - lg).max(axis=0) > 1e-6
    rows_p = (g == p).all(axis=0)
    assert off.sum() == bad and rows_p.sum() == at_p and not (rows_p & ~off).any()
    np.testing.assert_allclose(g[:, rows_p].sum(axis=0), p[:, rows_p].sum(axis=0), rtol=0, atol=1e-12)
    assert np.abs(g[:, rows_p].sum(axis=0)).min() > 0.99
    assert np.abs(lg.sum(axis=0)).max() <= 1e-9
    assert np.abs(g[:, ~off] - lg[:, ~off]).max() <= 1e-6


@pytest.mark.parametrize("T,K,L,scale,seed", LOST_MASS)
def test_lost_trellis_mass_shows_as_forward_backward_disagreement(T, K, L, scale, seed):
    """5000 frames, 300 labels, unaligned logits: the scaled trellis loses mass.  Its llForward and llBackward disagree
    by more than a nat, its loss is off the log-domain one by tens of nats, and nearly every gradient row is p.  The
    log-domain oracle's loss agrees with an independent log-domain forward pass, and its rows sum to 0."""
    p, seq = _utt(T, K, L, scale, seed)
    nll, g, skip, llb = ctc_oracle.ctc_loss_fb(p, seq)
    lnll, lg, lskip = ctc_oracle.ctc_loss_log(p, seq)
    assert not skip and not lskip
    assert abs(-nll - llb) > 1.0, (nll, llb)
    assert abs(nll - lnll) > 50.0, (nll, lnll)
    assert abs(lnll - _log_forward_nll(p, seq)) <= 1e-9 * lnll
    assert np.abs(lg.sum(axis=0)).max() <= 1e-9
    assert (np.abs(g - lg).max(axis=0) > 1e-6).sum() >= 4000
