"""GPU test of the blank-forced CTC kernel (ctcb_ctc_blankforce_loss_grad_f32) and of the best-path kernel
(ctcb_ctc_best_path_f32), against float64 oracles with element-wise bounds.

The reference is oracle.ctc_oracle.ctc_loss_blankforce_log (float64 log-sum-exp, no per-frame scaling) fed the float32
probabilities, or the float64 softmax of the float32 logits.  Per utterance: where the oracle skips, the kernel returns
skip = 1 and a zero gradient; elsewhere skip = 0, max |g - g_ref| <= GRAD_BOUND and |nll - nll_ref| / |nll_ref| <=
NLL_BOUND.  Rows at or beyond an utterance's T hold 0; the padding of a layout, the gaps of the gradient and a guard
after the workspace keep what was there.  The long-utterance cases are classified by the CPU oracles (the scaled one is
the reference's arithmetic) and each asserts its class.  Each case prints one JSON line with its errors and skips."""
import json

import numpy as np
import pytest

import recipes
from oracle import ctc_oracle
from recipes import Batch
from test_ctc_blankforce_cpu import EDGES, awkward_rows, np_best_path

pytestmark = pytest.mark.gpu
# 4x the largest errors measured on an H100 80GB HBM3 (DESIGN.md section 4)
GRAD_BOUND, NLL_BOUND = 3.6e-6, 2.4e-7
SENTINEL = 7.0
WS_GUARD = 4096
MAX_STATES = 1024
K_MAX = {1: 25565, 1024: 23008}        # 20 * max_states + 256 + 8 K <= 200 KiB of shared memory


def _ref(p, seq):
    """Log-domain result for float64 probabilities p (T x K)."""
    return ctc_oracle.ctc_loss_blankforce_log(np.asfortranarray(p.T), seq)


def _probs(b, u, T):
    x = b.x[u, :T]
    return x.astype(np.float64) if b.is_prob else recipes.softmax64(x)


def _launch(torch, b, max_states, lens=None, seqs=None, rc_expect=0):
    """Run the kernel on batch b; returns (nll, grad[B][Tmax][K], skip) after checking the buffers' gaps and guard."""
    from _ctcb import lib, check, ptr
    lens = b.lens if lens is None else lens
    seqs = b.seqs if seqs is None else seqs
    d_x = torch.from_numpy(b.flat(np.nan)).cuda()
    d_g = torch.from_numpy(np.full(b.n + 2, SENTINEL, dtype=np.float32)).cuda()
    flat = np.concatenate([np.asarray(s, np.int32) for s in seqs] + [np.zeros(1, np.int32)])
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int32)
    d_seq, d_off = torch.from_numpy(flat).cuda(), torch.from_numpy(off).cuda()
    d_T = torch.from_numpy(np.asarray(lens, np.int32)).cuda()
    need = lib.ctcb_ctc_blankforce_workspace_bytes(b.B, b.Tmax, max_states)
    ws = torch.full((need + WS_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    nll = torch.full((b.B,), -1.0, device="cuda")
    skip = torch.full((b.B,), -1, dtype=torch.int32, device="cuda")
    rc = lib.ctcb_ctc_blankforce_loss_grad_f32(d_x.data_ptr() + 4 * b.off, int(b.is_prob), b.us, b.fs, ptr(d_seq),
                                                ptr(d_off), ptr(d_T), b.B, b.Tmax, b.K, max_states,
                                                d_g.data_ptr() + 4 * b.off, ptr(nll), ptr(skip), ptr(ws), need,
                                                torch.cuda.current_stream().cuda_stream)
    if rc_expect:
        assert rc == rc_expect, rc
        return None
    check(rc)
    torch.cuda.synchronize()
    g = d_g.cpu().numpy()
    mask = np.ones(g.shape, bool)
    mask[b.idx] = False
    assert (g[mask] == SENTINEL).all(), "the kernel wrote outside the gradient's elements"
    assert (ws[need:] == 0xA5).all().item(), "the kernel wrote past its workspace"
    assert not np.isnan(g[b.idx]).any()
    return nll.cpu().numpy(), g[b.idx], skip.cpu().numpy()


def _check(torch, name, b, max_states, lens=None, expect_skip=None, classes=None):
    """Launch and compare every utterance with the log oracle; print one JSON line, then assert."""
    lens = b.lens if lens is None else lens
    nll, g, skip = _launch(torch, b, max_states, lens)
    gerr = nerr = 0.0
    problems, n_skip = [], 0
    for u in range(b.B):
        T = max(0, min(lens[u], b.Tmax))
        if (g[u, T:] != 0).any():
            problems.append("utterance %d: rows >= T written" % u)
        lnll, lg, lskip = _ref(_probs(b, u, T), b.seqs[u]) if T > 0 else (0.0, None, True)
        if skip[u] != int(lskip) or (expect_skip is not None and skip[u] != int(expect_skip[u])):
            problems.append("utterance %d: skip %d, oracle %d" % (u, skip[u], lskip))
            continue
        if lskip:
            n_skip += 1
            if g[u].any():
                problems.append("utterance %d: skipped with a gradient" % u)
            continue
        ge = float(np.abs(g[u, :T] - lg.T).max())
        if not np.isfinite(lnll):
            if nll[u] != lnll:
                problems.append("utterance %d: nll %g, oracle %g" % (u, nll[u], lnll))
            ne = 0.0
        else:
            ne = abs(float(nll[u]) - lnll) / abs(lnll)
        gerr, nerr = max(gerr, ge), max(nerr, ne)
    print(json.dumps(dict(bf=name, is_prob=b.is_prob, B=b.B, Tmax=b.Tmax, K=b.K, max_states=max_states,
                          grad_err=float(gerr), nll_err=float(nerr), skips=n_skip, classes=classes, problems=problems[:5])))
    assert not problems, problems
    assert gerr <= GRAD_BOUND and nerr <= NLL_BOUND, (gerr, nerr)
    return nll, g, skip


def _batch(utts, is_prob, layout="bt", fs_pad=0, off=0):
    """utts: (logits float32 T x K, seq).  Probability input is the float32 softmax of the logits."""
    Tmax, K = max(x.shape[0] for x, _ in utts), utts[0][0].shape[1]
    x = np.zeros((len(utts), max(Tmax, 1), K), np.float32)
    for u, (xu, _) in enumerate(utts):
        x[u, :xu.shape[0]] = recipes.softmax64(xu).astype(np.float32) if is_prob else xu
    return Batch(x, [xu.shape[0] for xu, _ in utts], [s for _, s in utts], is_prob=is_prob, layout=layout,
                 fs_pad=fs_pad, off=off)


def _states_utt(L, K, seed, T=None):
    rng = np.random.RandomState(seed)
    seq = (1 + rng.randint(K - 1, size=L)).astype(np.int32)
    seq[::2] = 0
    T = T or max(L + 24, 40)
    return (rng.randn(T, K) * 1.5).astype(np.float32), seq


TILING = [1, 2, 255, 256, 257, 511, 512, 513, 767, 768, 769, 1023, 1024]


@pytest.mark.parametrize("L", TILING)
def test_state_tiling_row_pitch_equals_L(L, cuda):
    """A thread owns states tid + 256 j, j = 0..3: every edge of that tiling, with max_states = L."""
    _check(cuda, "tiling-L%d" % L, _batch([_states_utt(L, 33, L)], False), L)


@pytest.mark.parametrize("is_prob", [False, True], ids=["logit", "prob"])
def test_state_tiling_wide_row_pitch(is_prob, cuda):
    """All the tiling edges in one batch at max_states = 1024: the row pitch is larger than L for all but the last."""
    _check(cuda, "tiling-all", _batch([_states_utt(L, 33, L, T=1100) for L in TILING], is_prob), MAX_STATES)


def test_trellis_edges(cuda):
    """T = 1, 2, L, T < L with and without alpha and beta meeting, the row-0 quirk, the reference's two
    zero-probability skips, an all-zero frame, a zero on the only path and exact zeros elsewhere (probability input)."""
    K = EDGES[0][1].shape[1]
    x = np.zeros((len(EDGES), max(e[1].shape[0] for e in EDGES), K), np.float32)
    for u, e in enumerate(EDGES):
        x[u, :e[1].shape[0]] = e[1]
    b = Batch(x, [e[1].shape[0] for e in EDGES], [e[2] for e in EDGES], is_prob=True)
    nll, g, skip = _check(cuda, "edges", b, max(len(e[2]) for e in EDGES), expect_skip=[e[3] for e in EDGES])
    names = [e[0] for e in EDGES]
    u = names.index("T_lt_L_apart")
    assert np.array_equal(g[u, :b.lens[u]], b.x[u, :b.lens[u]]) and np.isfinite(nll[u])
    assert nll[names.index("zero_first_state_frame0")] == np.inf


def test_T_per_utt_beyond_Tmax_and_zero(cuda):
    utts = [_states_utt(9, 12, s, T=30) for s in range(4)]
    b = _batch(utts, False)
    lens = [30, 45, 0, 17]                                  # 45 > Tmax: the kernel reads Tmax frames
    nll, g, skip = _check(cuda, "T_per_utt", b, 9, lens=lens, expect_skip=[0, 0, 1, 0])
    assert not g[2].any()


# (T, labels, logit scale, seed, aligned, class): recipes.bf_utt at K = 40
RANGE = [(1500, 150, 2.0, 1, False, "in"), (1500, 150, 3.0, 1, False, "in"),
         (3000, 300, 2.0, 1, False, "underflow"), (3000, 300, 3.0, 3, False, "underflow"),
         (5000, 300, 2.0, 1, False, "lost"), (5000, 300, 3.0, 3, False, "lost"),
         (1500, 150, 3.0, 1, True, "in"), (5000, 300, 3.0, 3, True, "in")]


def _range_utt(T, nlab, scale, seed, aligned):
    x, seq = recipes.bf_utt(T, 40, nlab, scale, seed)
    if aligned:                                             # outputs that follow the states in order
        x[np.arange(T), seq[np.arange(T) * len(seq) // T]] += 6.0
    return x, seq


def _classify(p, seq):
    nll, g, skip = ctc_oracle.ctc_loss_blankforce(np.asfortranarray(p.T), seq)
    lnll, lg, lskip = _ref(p, seq)
    assert not skip and not lskip
    if abs(nll - lnll) > 1.0:
        return "lost"
    if abs(nll - lnll) <= 1e-8 * lnll:
        return "in" if np.abs(g - lg).max() <= 1e-6 else "underflow"
    return "between"


@pytest.mark.parametrize("is_prob", [False, True], ids=["logit", "prob"])
@pytest.mark.parametrize("case", RANGE, ids=lambda c: "T%d-L%d-s%g-seed%d-%s%s" % (
    c[0], 2 * c[1] + 1, c[2], c[3], "aligned-" if c[4] else "", c[5]))
def test_long_utterance(case, is_prob, cuda):
    """In range, underflowing and mass-losing utterances: the kernel computes every one of them correctly."""
    b = _batch([_range_utt(*case[:5])], is_prob)
    cls = _classify(_probs(b, 0, b.lens[0]), b.seqs[0])
    assert cls == case[5], (case, cls)
    _check(cuda, "range", b, len(b.seqs[0]), expect_skip=[0], classes=[cls])


@pytest.mark.parametrize("layout,fs_pad,off", [("tb", 0, 0), ("bt", 3, 0), ("bt", 0, 5), ("tb", 1, 3)],
                         ids=["time-major", "padded", "offset", "time-major-padded-offset"])
def test_layouts(layout, fs_pad, off, cuda):
    """Ragged utterances in the BRNN's time-major layout, a padded frame stride and a base offset; the gaps hold NaN."""
    rng = np.random.RandomState(3)
    utts = [_states_utt(int(L), 29, 100 + i, T=int(T)) for i, (L, T) in
            enumerate(zip(rng.randint(1, 300, size=7), rng.randint(1, 400, size=7)))]
    _check(cuda, "layout-%s-%d-%d" % (layout, fs_pad, off), _batch(utts, False, layout, fs_pad, off), 300)


def test_ragged_batch_beyond_one_wave(cuda):
    """1200 short utterances: more CTAs than one wave of the H100 holds at this shared-memory size."""
    rng = np.random.RandomState(9)
    utts = [_states_utt(int(L), 20, 1000 + i, T=int(T)) for i, (L, T) in
            enumerate(zip(rng.randint(1, 42, size=1200), rng.randint(20, 61, size=1200)))]
    _check(cuda, "ragged-1200", _batch(utts, False, "tb"), 41)


@pytest.mark.parametrize("K", [2, 31, 32, 33, 64, 1000])
def test_vocabulary_sizes(K, cuda):
    utts = [_states_utt(L, K, K + L, T=T) for L, T in ((1, 5), (7, 40), (61, 90), (200, 260))]
    _check(cuda, "K%d" % K, _batch(utts, False), 200)


@pytest.mark.parametrize("max_states", [1, 1024])
def test_largest_vocabulary(max_states, cuda):
    """The largest K the launcher accepts at max_states = 1 and 1024 runs; one more is CTCB_EINVAL."""
    K = K_MAX[max_states]
    rng = np.random.RandomState(max_states)
    T = 6 if max_states == 1 else 1040
    seq = (1 + rng.randint(K - 1, size=max_states)).astype(np.int32)
    x = (rng.randn(1, T, K) * 2).astype(np.float32)
    _check(cuda, "K-max", Batch(x, [T], [seq]), max_states)
    x1 = np.zeros((1, 2, K + 1), np.float32)
    assert _launch(cuda, Batch(x1, [2], [seq]), max_states, rc_expect=-1) is None


def test_contract_violations_skip_without_touching_the_batch(cuda):
    """An empty sequence, more states than max_states and a label outside [0, K): skip = 1 with a zero gradient, and
    the other utterances are the same bits as in a batch without them."""
    K, ms = 17, 40
    good = [_states_utt(L, K, 50 + L, T=60) for L in (39, 40, 21)]
    over = _states_utt(ms + 9, K, 7, T=60)
    neg = _states_utt(15, K, 8, T=60)
    neg[1][3] = -1
    big = _states_utt(15, K, 9, T=60)
    big[1][6] = K
    empty = (good[0][0], np.zeros(0, np.int32))
    mixed = [good[0], empty, over, good[1], neg, big, good[2]]
    nll, g, skip = _launch(cuda, _batch(mixed, False), ms)
    assert skip.tolist() == [0, 1, 1, 0, 1, 1, 0]
    assert not g[[1, 2, 4, 5]].any()
    nll0, g0, skip0 = _launch(cuda, _batch(good, False), ms)
    for u, v in ((0, 0), (3, 1), (6, 2)):
        assert nll[u].tobytes() == nll0[v].tobytes() and g[u].tobytes() == g0[v].tobytes() and skip0[v] == 0
    print(json.dumps(dict(bf="contract", skips=skip.tolist())))


def test_same_bits_twice(cuda):
    b = _batch([_range_utt(3000, 300, 3.0, 3, False)] + [_states_utt(L, 40, L) for L in (5, 300, 601)], False)
    r1, r2 = _launch(cuda, b, 601), _launch(cuda, b, 601)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(r1, r2))


# ------------------------------------------------------------------------------------------------ best path
def _best_path(torch, rows, lens, blank, drop):
    """rows: B x Tmax x K float32; returns per utterance (hyp, align)."""
    from _ctcb import lib, check, ptr
    B, Tmax, K = rows.shape
    d = torch.from_numpy(rows).cuda()
    tl = torch.from_numpy(np.asarray(lens, np.int32)).cuda()
    hyp = torch.full((B * Tmax,), -7, dtype=torch.int32, device="cuda")
    ali = torch.full((B * Tmax,), -7, dtype=torch.int32, device="cuda")
    n = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    check(lib.ctcb_ctc_best_path_f32(ptr(d), Tmax * K, K, ptr(tl), B, Tmax, K, blank, drop, ptr(hyp), ptr(ali), ptr(n),
                                     torch.cuda.current_stream().cuda_stream))
    hyp, ali, n = hyp.cpu().numpy().reshape(B, Tmax), ali.cpu().numpy().reshape(B, Tmax), n.cpu().numpy()
    return [(hyp[u, :n[u]].tolist(), ali[u, :n[u]].tolist()) for u in range(B)]


@pytest.mark.parametrize("drop", [0, 1], ids=["no-filter", "filter-1-2-8"])
@pytest.mark.parametrize("K", [5, 31, 32, 33, 70])
def test_best_path_follows_np_argmax(K, drop, cuda):
    """Ties across lanes, NaN at index 0 and inside a row, all-NaN and all -inf rows, +inf, runs of repeats and ragged
    T_per_utt, with the blank at 0, in the middle and at K - 1."""
    B, Tmax = 6, 150
    rows = np.ascontiguousarray(np.stack([awkward_rows(K, Tmax, 31 * K + u).T for u in range(B)]))
    lens = [150, 1, 0, 77, 149, 200]
    for blank in (0, K // 2, K - 1):
        got = _best_path(cuda, rows, lens, blank, drop)
        with np.errstate(invalid="ignore"):
            want = [np_best_path(rows[u, :min(lens[u], Tmax)].T.astype(np.float64), blank, bool(drop)) for u in range(B)]
        assert got == want
        assert all(0 <= h < K for hyp, _ in got for h in hyp)
