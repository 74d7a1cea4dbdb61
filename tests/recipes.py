"""Deterministic input recipes shared by the golden generator and the tests.

All follow the reference's own eyeball tests (seed 33, legacy np.random streams):
  time_trials : ctc/time_trials.py:13-25  (K=40, |l|=125, T=1200, peaked probs)
  ctc_py      : ctc/ctc.py:143-152        (K=62, |l|=54, T=453, logits ~ N(0,1))
  c1          : BASELINE.json configs[0]                  (T=200, K=62, |l|=30)
  rnnetcpu    : ctc_fast/debug-utils/rnnetcpu.py:181-193 (D=20,T=10,K=6,H=30,N=3,tl=2)
"""
import numpy as np
import pytest


@pytest.fixture
def knobs():
    """knobs(name, value) sets a planner knob in this process (ctcb_debug_set_knob, environment syntax); every knob it
    set is restored to what the environment said when the test ends, pass or fail.  A test module that uses it imports
    it: `from recipes import knobs`."""
    from _ctcb import lib, check
    touched = set()

    def set_(name, value):
        touched.add(name)
        check(lib.ctcb_debug_set_knob(name.encode(), value.encode()))
    yield set_
    for name in touched:
        check(lib.ctcb_debug_set_knob(name.encode(), None))


def softmax_cols(x):
    x = x - x.max(axis=0)
    e = np.exp(x)
    return e / e.sum(axis=0)


def time_trials():
    np.random.seed(33)
    numPhones, seqLen, uttLen = 40, 125, 1200
    seq = np.floor(np.random.rand(seqLen) * numPhones).astype(np.int32)
    params = np.random.randn(numPhones, uttLen)
    params[seq, np.arange(seqLen)] = 3
    params[0, seqLen:] = 3
    params = np.exp(params)
    params = params / np.sum(params, axis=0)
    return params, seq


def ctc_py():
    np.random.seed(33)
    numPhones, seqLen, uttLen = 62, 54, 453
    seq = np.floor(np.random.rand(seqLen, 1) * numPhones).astype(np.int32).reshape(-1)
    logits = np.random.randn(numPhones, uttLen)
    return logits, seq


def synth_ctc(T, K, nlab, seed=33):
    """Sweep-style case: logits ~ N(0,1), labels uniform over non-blank (ctc/gradcheck.py:68-69)."""
    rng = np.random.RandomState(seed + 1000003 * T + 1009 * K + nlab)
    logits = rng.randn(K, T)
    seq = (1 + np.floor(rng.rand(nlab) * (K - 1))).astype(np.int32)
    return logits, seq


CTC_CASES = {
    # name: (T, K, |l|)
    "c1": (200, 62, 30),
    "sweep_100_10_32": (100, 32, 10),
    "sweep_500_100_62": (500, 62, 100),
    "sweep_500_300_128_infeasible_len": (100, 128, 300),
    "wsj_800_100_32": (800, 32, 100),
    "swbd_1500_150_35": (1500, 35, 150),
    "long_2000_300_128": (2000, 128, 300),
    "repeat_heavy": (64, 8, 31),
    "single_label": (5, 4, 1),
    "T_equals_L": (12, 9, 12),
    "T_equals_L_feasible": (12, 16, 12),
}


def ctc_case(name):
    """Returns (probs float32 K x T, seq int32).  probs are float32-rounded softmax outputs, which is
    what the reference's CTC receives from the GPU (brnnet.py:170-175)."""
    if name == "time_trials":
        p, s = time_trials()
        return p.astype(np.float32), s
    if name == "ctc_py":
        l, s = ctc_py()
        return softmax_cols(l).astype(np.float32), s
    T, K, nlab = CTC_CASES[name]
    logits, seq = synth_ctc(T, K, nlab)
    if name == "repeat_heavy":
        seq = (1 + (np.arange(nlab) // 3) % (K - 1)).astype(np.int32)   # runs of repeated labels
    if name == "T_equals_L_feasible":
        seq = (1 + np.arange(nlab)).astype(np.int32)                    # all distinct: exactly one path
    return softmax_cols(logits).astype(np.float32), seq


ALL_CTC = ["time_trials", "ctc_py"] + list(CTC_CASES)


def golden_stride(K, T):
    """Golden gradients of the big cases are stored for every 8th frame only (fixtures stay small)."""
    return 1 if K * T <= 50000 else 8


def rnnetcpu():
    """Data, labels and an oracle-initialised parameter stack for the reference's CPU BRNN self-test."""
    np.random.seed(33)
    data = np.random.randn(20, 10)
    labels = np.arange(3).astype(np.int32)
    return dict(inputDim=20, outputDim=6, layerSize=30, numLayers=3, temporalLayer=2, maxBatch=10), data, labels


def synth_batch(inputDim, outputDim, lens, nlabs, seed=33):
    """Features randn(D,T) float32 (rnnetcpu.py:189), labels uniform over non-blank."""
    rng = np.random.RandomState(seed)
    datas = [rng.randn(inputDim, T).astype(np.float32) for T in lens]
    labels = [(1 + np.floor(rng.rand(n) * (outputDim - 1))).astype(np.int32) for n in nlabs]
    return datas, labels


# ---- blank-forced CTC (ctc_fast_blankforce.pyx): the sequence carries its blanks ---------------------
BF_CASES = {
    # name: (T, K, number of non-blank labels)
    "bf_c1": (200, 62, 30),
    "bf_small": (10, 6, 3),
    "bf_wsj": (800, 32, 100),
    "bf_long": (1500, 35, 300),
    "bf_T_less_than_L": (8, 10, 6),          # no exception in the reference: absum == 0 -> grad = probs
    "bf_no_leading_blank": (50, 20, 10),     # seq[0] != 0 exercises the row-0 quirk (:49)
    "bf_one_state": (7, 5, 0),
    "bf_peaked": (400, 40, 60),
}


def bf_case(name):
    """Returns (probs float32 K x T, seq int32 with blanks interleaved: 0 l1 0 l2 ... 0)."""
    T, K, nlab = BF_CASES[name]
    logits, lab = synth_ctc(T, K, nlab, seed=77)
    if name == "bf_peaked":
        logits = logits * 4.0
    seq = np.zeros(2 * nlab + 1, dtype=np.int32)
    seq[1::2] = lab
    if name == "bf_no_leading_blank":
        seq = seq[1:].copy()
    return softmax_cols(logits).astype(np.float32), seq


ALL_BF = list(BF_CASES)


def bf_utt(T, K, nlab, scale, seed):
    """One blank-forced utterance: float32 logits (T x K) ~ N(0, scale^2) and 0 l1 0 l2 ... 0 with nlab labels drawn
    uniformly from 1..K-1 (2 nlab + 1 states)."""
    rng = np.random.RandomState(seed)
    x = (rng.randn(T, K) * scale).astype(np.float32)
    seq = np.zeros(2 * nlab + 1, dtype=np.int32)
    seq[1::2] = 1 + rng.randint(K - 1, size=nlab)
    return x, seq


RNN_VARIANTS = (("uni", dict(temporalLayer=2, unidirectional=True)), ("dnn", dict(temporalLayer=-1)))


def rnn_variant_batch():
    return synth_batch(13, 11, [30, 41, 12, 41], [7, 11, 3, 15], seed=11)


def rnn_variant_net(cls, tag, **extra):
    """The uni-directional (nnets/rnnet.py) / feed-forward (nnets/nnet.py) golden nets: D=13, K=11, H=64, N=3."""
    kw = dict(RNN_VARIANTS)[tag]
    np.random.seed(9)
    nn = cls(13, 11, 64, 3, 41, **dict(kw, **extra))
    nn.initParams()
    return nn


def rnn_variant_perturb(stack, tag):
    """Host-side edits of the freshly initialised stack (list of [w, b] arrays) that the golden nets carry."""
    for w, b in stack[:3]:
        b += 0.05
    if tag == "uni":
        stack[1][1] += 4.0          # some units reach the 20.0 clip (rnnet.py:32,113-116)
        stack[-1][0] *= 1.2


# ---- randomised shapes on which the C restatements are pinned to the compiled reference modules ----------------
def random_ctc_cases():
    """300 random (K, T, |l|) cases incl. T = 1, T = |l|, T < |l|, heavy label repetition and peaked distributions."""
    rng = np.random.RandomState(2024)
    for case in range(300):
        K = int(rng.randint(2, 40))
        T = int(rng.choice([1, 2, 3, 5, 8, 17, 40, 90]))
        nlab = int(rng.randint(1, max(2, min(T + 3, 25))))
        scale = float(rng.choice([0.5, 1.0, 4.0, 12.0]))
        probs = softmax_cols(rng.randn(K, T) * scale).astype(np.float32).astype(np.float64)
        if rng.rand() < 0.3:
            seq = np.full(nlab, 1 + rng.randint(K - 1), dtype=np.int32)           # one label repeated
        else:
            seq = (1 + rng.randint(0, K - 1, size=nlab)).astype(np.int32)
        yield np.asfortranarray(probs), seq


def random_bf_cases():
    """200 random blank-forced cases, most with the usual interleaved blanks."""
    rng = np.random.RandomState(77)
    for case in range(200):
        K = int(rng.randint(2, 30))
        T = int(rng.choice([1, 2, 4, 9, 33, 70]))
        L = int(rng.randint(1, 20))
        probs = softmax_cols(rng.randn(K, T) * float(rng.choice([1.0, 5.0]))).astype(np.float32).astype(np.float64)
        seq = rng.randint(0, K, size=L).astype(np.int32)
        if rng.rand() < 0.7:
            seq[::2] = 0                                                           # the usual interleaved blanks
        yield np.asfortranarray(probs), seq


# ---- batches for the GPU CTC kernel (tests/test_ctc_plans_gpu.py, tests/test_ctc_range_gpu.py) -------------------
class Batch:
    """B utterances with element (u, t, k) at off + u*us + t*fs + k of one float32 buffer; gaps hold NaN."""

    def __init__(self, x, lens, seqs, is_prob=False, blank=0, layout="bt", fs_pad=0, off=0):
        B, Tmax, K = x.shape
        self.x, self.lens, self.seqs, self.is_prob, self.blank = x, list(lens), list(seqs), is_prob, blank
        self.B, self.Tmax, self.K = B, Tmax, K
        if layout == "bt":
            self.fs = K + fs_pad
            self.us = Tmax * self.fs
        else:                       # time-major, as the BRNN lays its logits out: [Tmax][B][K]
            self.us = K + fs_pad
            self.fs = B * self.us
        self.off = off
        self.n = off + (B - 1) * self.us + (Tmax - 1) * self.fs + K
        self.idx = (off + np.arange(B)[:, None, None] * self.us + np.arange(Tmax)[None, :, None] * self.fs
                    + np.arange(K)[None, None, :])

    def flat(self, fill):
        buf = np.full(self.n + 2, fill, dtype=np.float32)
        buf[self.idx] = self.x
        return buf


def softmax64(x):
    """Row softmax in float64 of an (n, K) array."""
    x = x.astype(np.float64)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def ctc_labels(rng, n, K, blank, repeats=0.0):
    """n labels over the non-blank classes; `repeats`: probability that a label repeats its predecessor."""
    cls = np.array([k for k in range(K) if k != blank])
    s = cls[rng.randint(0, len(cls), size=n)]
    for i in range(1, n):
        if rng.rand() < repeats:
            s[i] = s[i - 1]
    return s.astype(np.int32)


def ctc_batch(B, T, K, L, seed, is_prob=False, blank=0, ragged=True, scale=2.0, repeats=0.1, **layout):
    """Logits ~ N(0, scale^2) (or their float32 softmax, is_prob), labels from ctc_labels; ragged: the first utterance
    is the longest (T frames, L labels), the others mostly feasible."""
    rng = np.random.RandomState(seed)
    x = (rng.randn(B, T, K) * scale).astype(np.float32)
    lens = [T] * B
    nl = [L] * B
    if ragged and B > 1:
        lens = [T] + [int(v) for v in rng.randint(max(1, 3 * T // 4), T + 1, size=B - 1)]
        nl = [L] + [int(rng.randint(max(1, L // 2), max(max(1, L // 2), min(L, 4 * t // 5)) + 1)) for t in lens[1:]]
    seqs = [ctc_labels(rng, nl[u], K, blank, repeats=repeats) for u in range(B)]
    if is_prob:
        x = softmax64(x.reshape(B * T, K)).reshape(B, T, K).astype(np.float32)
    return Batch(x, lens, seqs, is_prob=is_prob, blank=blank, **layout)


def ctc_trellis_edges(K=12, seed=5):
    """(T, labels) of one utterance per edge of the trellis, to be run as one batch."""
    rng = np.random.RandomState(seed)
    rows = []
    distinct = lambda n: (1 + rng.permutation(K - 1)[:n]).astype(np.int32)

    def add(T, s):
        rows.append((T, np.asarray(s, np.int32)))
    add(1, [3]); add(2, [3]); add(3, [3, 4])                         # T = 1, 2, 3
    add(1, [2, 5])                                                   # one frame, two labels: finite, see short_utt_nll
    add(5, distinct(5))                                              # T = |l|, distinct: one path
    add(5, [1, 2, 2, 3, 4])                                          # T = |l| with a repeat: infeasible -> skip
    add(6, [1, 2, 2, 3, 4])                                          # T = |l| + repeats: one path again
    add(10, [1, 1, 1, 2, 2, 2])                                      # T = |l| + repeats, runs
    add(4, [5, 6, 7, 8, 9, 10])                                      # T < |l|: inf
    add(90, [7] * 31)                                                # a run of repeats across lane boundaries
    add(80, np.repeat(distinct(4), 8)[:30])                          # runs crossing pair i = lane * P + j
    add(70, distinct(11))
    return rows


def digest(a):
    """SHA-256 of a float64 array's values (row-major, every NaN canonical) as 32 uint8: a stored stand-in for a
    bit-exact comparison with an array that is too large to keep."""
    import hashlib
    a = np.ascontiguousarray(a, dtype=np.float64)
    a = np.where(np.isnan(a), np.nan, a)
    return np.frombuffer(hashlib.sha256(a.tobytes()).digest(), dtype=np.uint8)
