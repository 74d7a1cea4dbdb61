"""GPU unit test of the CTC loss + gradient (ctcb_ctc_loss_grad_f32) on every plan its planner can choose, against the
float64 C restatement of ctc_fast.pyx (oracle.ctc_oracle, pinned bit-exact to the reference).

The planner (select_ctc, csrc/ctc.cu) picks one of four kernel organisations -- the frame-parallel kernel (par), the two
warps meeting in the middle (pair), one warp per utterance with on-chip checkpoints (ckpt) or with the trellis spilled
(warp) -- at 1, 2, 4, 8 or 16 (blank, label) pairs per lane, with 8- or 16-frame tiles, one or two tile buffers, and
4- or 8-byte tile copies and stores (vec2).  Every case names the plan it targets and checks it with ctcb_debug_ctc_plan
before launching, so no case passes on a plan it did not mean to test; forced organisations are set in process with
the CTCB_CTC knob (ctcb_debug_set_knob) and reset by a fixture.

The reference sees the kernel's inputs: the float32 probabilities as they are, or the float64 softmax of the float32
logits.  The bounds are element-wise: max |g - g_ref| over every valid (t, k) of every compared utterance, and
|nll - nll_ref| / |nll_ref| per utterance; skip flags equal; padded frames and skipped utterances exactly 0; T < |l|
gives inf with the reference's gradient; nothing outside the gradient's (u, t < Tmax, k < K) elements is written.
Each case prints its plan, errors and bounds as one JSON line (shown with pytest -s)."""
import ctypes
import json
import time

import numpy as np
import pytest

from oracle import ctc_oracle
from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
H100_SMS = 132             # the plans below are laid out for the 132-SM H100 SXM; other parts skip a plan they cannot reach
KERNELS = ("par", "pair", "ckpt", "warp")
FIELDS = ("kernel", "P", "th", "nbuf", "warps", "vec2", "Kp", "smem_kb")
# Bounds per organisation (max |g - g_ref|, |nll - nll_ref| / |nll_ref|), at most 4x the largest error measured on an H100
# 80GB HBM3 (power limit 700 W) over the cases of this file: par 4.7e-7 / 7.3e-8, pair 1.17e-6 / 9.9e-8, ckpt 5.3e-7 /
# 8.1e-8, warp 1.07e-6 / 1.11e-7 (DESIGN.md section 4).  The gradient error comes from the 2^-24 quantisation of the lane
# sums and the 2^30 fixed-point occupancies; the NLL error from the float32 sum of log Z.
BOUNDS = {"par": (1.7e-6, 2.9e-7), "pair": (4.6e-6, 3.9e-7), "ckpt": (2.1e-6, 3.2e-7), "warp": (4.2e-6, 4.4e-7)}
SENTINEL = 7.0             # fills the gradient buffer's gaps (odd strides, offsets): the kernel must leave it alone


# ------------------------------------------------------------------------------------------------ plans
def _plan(B, Tmax, K, L, acts=256, grad=256, us=None, fs=None):
    """(rc, plan dict) of ctcb_debug_ctc_plan; acts / grad are addresses (only their alignment matters)."""
    from _ctcb import lib
    out = (ctypes.c_int32 * 8)()
    rc = lib.ctcb_debug_ctc_plan(B, Tmax, K, L, acts, grad, Tmax * K if us is None else us, K if fs is None else fs,
                                 out)
    if rc != 0:
        return rc, None
    plan = dict(zip(FIELDS, list(out)))
    plan["kernel"] = KERNELS[plan["kernel"]]
    return rc, plan


def _check_plan(plan, expect, torch, what):
    wrong = {k: (v, plan.get(k)) for k, v in expect.items() if plan.get(k) != v}
    if wrong:
        msg = "%s: planned %s, this case targets %s" % (what, plan, expect)
        if torch.cuda.get_device_properties(0).multi_processor_count != H100_SMS:
            pytest.skip("plan not reachable on this device: " + msg)
        pytest.fail(msg)


@pytest.fixture
def force(knobs, cuda):
    """force(name) sets the organisation (auto, warp, pair, par, ckpt) in this process, overriding the environment's
    CTCB_CTC, which is in effect again afterwards."""
    def set_(name):
        knobs("CTCB_CTC", name)
    set_("auto")
    return set_


# ------------------------------------------------------------------------------------------------ one batch
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


def _run(torch, b, max_labels=None, plan_expect=None, what="", check_rc=True):
    """Launch ctcb_ctc_loss_grad_f32 on batch b; returns (plan, nll, grad[B][Tmax][K], skip, gaps of the gradient)."""
    import _ctcb
    from _ctcb import lib, check, ptr
    L = max(len(s) for s in b.seqs) if max_labels is None else max_labels
    # the buffers start 256-byte aligned; `off` floats in front make the base 4- but not 8-byte aligned when odd
    d_x = torch.from_numpy(b.flat(np.nan)).cuda()
    d_g = torch.from_numpy(np.full(b.n + 2, SENTINEL, dtype=np.float32)).cuda()
    x0, g0 = d_x.data_ptr() + 4 * b.off, d_g.data_ptr() + 4 * b.off
    rc, plan = _plan(b.B, b.Tmax, b.K, L, x0, g0, b.us, b.fs)
    if plan_expect is not None:
        assert rc == 0, _ctcb.lib.ctcb_last_error()
        _check_plan(plan, plan_expect, torch, what)
    lab = np.concatenate([np.asarray(s, np.int32) for s in b.seqs] + [np.zeros(1, np.int32)])
    off = np.concatenate([[0], np.cumsum([len(s) for s in b.seqs])]).astype(np.int32)
    d_lab, d_off = torch.from_numpy(lab).cuda(), torch.from_numpy(off).cuda()
    d_len = torch.tensor(b.lens, dtype=torch.int32).cuda()
    nll = torch.full((b.B,), -1.0, device="cuda")
    skip = torch.full((b.B,), -1, dtype=torch.int32, device="cuda")
    nws = int(lib.ctcb_ctc_workspace_bytes(b.B, b.Tmax, L))
    ws = torch.empty(max(nws, 8), dtype=torch.uint8, device="cuda")
    r = lib.ctcb_ctc_loss_grad_f32(x0, int(b.is_prob), b.us, b.fs, ptr(d_lab), ptr(d_off), ptr(d_len), b.B, b.Tmax,
                                   b.K, L, b.blank, g0, ptr(nll), ptr(skip), ptr(ws), nws, _ctcb.current_stream())
    if not check_rc:
        return r, plan
    check(r)
    torch.cuda.synchronize()
    g = d_g.cpu().numpy()
    mask = np.ones(g.shape, bool)
    mask[b.idx] = False
    return plan, nll.cpu().numpy().astype(np.float64), g[b.idx].astype(np.float64), skip.cpu().numpy(), g[mask]


def _softmax64(x):
    x = x.astype(np.float64)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def _compare(b, res, utts=None):
    """Per-utterance comparison with the oracle; returns (max grad error, max nll error, counts).  Asserts the exact
    properties (skip flags, zeros, inf, untouched gaps) as it goes."""
    plan, nll, g, skip, gaps = res
    assert (gaps == SENTINEL).all(), "the kernel wrote outside the gradient's elements"
    assert set(np.unique(skip)) <= {0, 1}, "skip flags not written"
    gerr = nerr = 0.0
    n = dict(ok=0, skip=0, inf=0)
    for u in (range(b.B) if utts is None else utts):
        T = min(b.lens[u], b.Tmax)
        assert not g[u, max(T, 0):].any(), "padded frames of utterance %d carry gradient" % u
        if T <= 0:
            assert skip[u] == 1 and not g[u].any(), u
            n["skip"] += 1
            continue
        xu = b.x[u, :T]
        p = xu.astype(np.float64) if b.is_prob else _softmax64(xu)
        o_nll, o_g, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(p.T), np.asarray(b.seqs[u], np.int32), b.blank)
        assert bool(skip[u]) == o_skip, (u, skip[u], o_skip, nll[u], o_nll)
        if o_skip:
            assert not g[u].any(), "skipped utterance %d has a gradient" % u
            n["skip"] += 1
            continue
        gerr = max(gerr, float(np.abs(g[u, :T] - o_g.T).max()))
        if np.isinf(o_nll):
            assert np.isinf(nll[u]) and nll[u] > 0, (u, nll[u])
            n["inf"] += 1
            continue
        nerr = max(nerr, abs(nll[u] - o_nll) / abs(o_nll))
        n["ok"] += 1
    return gerr, nerr, n


def _report(name, plan, gerr, nerr, n, t0, **extra):
    gb, nb = BOUNDS[plan["kernel"]]
    print(json.dumps(dict(ctc=name, plan=plan, grad_err=gerr, nll_err=nerr, grad_bound=gb, nll_bound=nb,
                          utterances=n, seconds=round(time.time() - t0, 2), **extra)))
    assert gerr <= gb, (name, gerr, gb)
    assert nerr <= nb, (name, nerr, nb)


# ------------------------------------------------------------------------------------------------ batch builders
def _labels(rng, n, K, blank, T=None, repeats=0.0):
    """n labels over the non-blank classes; `repeats`: probability that a label repeats its predecessor."""
    cls = np.array([k for k in range(K) if k != blank])
    s = cls[rng.randint(0, len(cls), size=n)]
    for i in range(1, n):
        if rng.rand() < repeats:
            s[i] = s[i - 1]
    return s.astype(np.int32)


def _make(B, T, K, L, seed, is_prob=False, blank=0, ragged=True, scale=2.0, repeats=0.1, **layout):
    rng = np.random.RandomState(seed)
    x = (rng.randn(B, T, K) * scale).astype(np.float32)
    lens = [T] * B
    nl = [L] * B
    if ragged and B > 1:                # the first utterance is the longest; the others mostly feasible
        lens = [T] + [int(v) for v in rng.randint(max(1, 3 * T // 4), T + 1, size=B - 1)]
        nl = [L] + [int(rng.randint(max(1, L // 2), max(max(1, L // 2), min(L, 4 * t // 5)) + 1)) for t in lens[1:]]
    seqs = [_labels(rng, nl[u], K, blank, repeats=repeats) for u in range(B)]
    if is_prob:
        x = _softmax64(x.reshape(B * T, K)).reshape(B, T, K).astype(np.float32)
    return Batch(x, lens, seqs, is_prob=is_prob, blank=blank, **layout)


def _case(torch, force, name, b, expect, forced="auto", utts=None, max_labels=None):
    t0 = time.time()
    force(forced)
    res = _run(torch, b, max_labels, expect, name)
    gerr, nerr, n = _compare(b, res, utts)
    _report(name, res[0], gerr, nerr, n, t0, forced=forced, B=b.B, Tmax=b.Tmax, K=b.K, is_prob=b.is_prob)
    assert n["ok"] > 0
    return res


# ------------------------------------------------------------------------------------------------ every organisation
# x every P it supports, label counts at the tiling edges (P = 1 holds at most 31 labels, 2: 63, 4: 127, 8: 255, 16: 511)
def _org_cases():
    edges = {1: (31,), 2: (32, 63), 4: (64, 127), 8: (128, 255), 16: (256, 511)}
    return [pytest.param(kern, forced, B, P, L, id="%s-P%d-L%d" % (kern, P, L))
            for kern, forced, B in (("par", "auto", 4), ("pair", "auto", 140), ("ckpt", "ckpt", 24), ("warp", "warp", 24))
            for P, labs in edges.items() if not (kern == "ckpt" and P > 4) for L in labs]


@pytest.mark.parametrize("kern,forced,B,P,L", _org_cases())
def test_organisation_and_pairs_per_lane(kern, forced, B, P, L, cuda, force):
    K = 40
    T = L + L // 4 + 8 + (L % 7)
    b = _make(B, T, K, L, seed=1000 * P + L + B)
    for u in range(1, B, 5):            # some utterances ragged below their label count: T < |l| -> inf
        b.lens[u] = max(1, len(b.seqs[u]) - 3)
    _case(cuda, force, "org-%s-P%d-L%d" % (kern, P, L), b, dict(kernel=kern, P=P), forced)


# ------------------------------------------------------------------------------------------------ warp-kernel tiles
@pytest.mark.parametrize("name,L,K,forced,th,nbuf", [
    ("warp-16x2", 40, 40, "warp", 16, 2),
    ("warp-16x1-P4", 100, 40, "warp", 16, 1),      # the checkpoint kernel takes P = 4 at this K automatically
    ("warp-16x1-P8", 200, 40, "auto", 16, 1),
    ("warp-8x1-P1", 20, 80, "auto", 8, 1),         # K > 64 P: the spill is cheaper than the checkpoints
    ("warp-8x1-P2", 50, 40, "warp", 8, 1),
])
def test_warp_kernel_tiles(name, L, K, forced, th, nbuf, cuda, force):
    """One tile buffer needs B >= 16 x SMs (2112 on an H100); short utterances keep that cheap.  Every utterance is
    compared with the oracle."""
    B = 16 * H100_SMS + 88 if nbuf == 1 else 64
    T = L + L // 4 + 6
    b = _make(B, T, K, L, seed=len(name) + L, repeats=0.2)
    _case(cuda, force, name, b, dict(kernel="warp", th=th, nbuf=nbuf), forced)


# ------------------------------------------------------------------------------------------------ vec2 paths
def _vec2_cases():
    cases = []
    for K in (30, 31, 62, 63, 130, 131):           # K <= 32, 33..64, > 64 for the 8-byte and the 4-byte paths
        for is_prob in (False, True):
            cases.append(pytest.param(K, is_prob, 0, 0, K % 2 == 0, id="K%d-%s" % (K, "prob" if is_prob else "logit")))
    for K in (30, 62, 130):
        cases.append(pytest.param(K, False, 1, 0, False, id="K%d-odd-frame-stride" % K))
        cases.append(pytest.param(K, True, 0, 1, False, id="K%d-base-plus-one-float" % K))
    return cases


@pytest.mark.parametrize("K,is_prob,fs_pad,off,vec2", _vec2_cases())
@pytest.mark.parametrize("kern,forced,B", [("par", "auto", 3), ("ckpt", "ckpt", 6), ("warp", "warp", 6)])
def test_vec2_paths(kern, forced, B, K, is_prob, fs_pad, off, vec2, cuda, force):
    L = 25
    b = _make(B, 61, K, L, seed=K + 7 * fs_pad + 11 * off + int(is_prob), is_prob=is_prob, fs_pad=fs_pad, off=off)
    _case(cuda, force, "vec2-%s-K%d-fs%d-off%d-%s" % (kern, K, fs_pad, off, is_prob), b,
          dict(kernel=kern, vec2=int(vec2)), forced)


# ------------------------------------------------------------------------------------------------ K limits
def _scan(B, L, Ks, forced, force):
    force(forced)
    return {K: _plan(B, 40, K, L) for K in Ks}


# The limits, from select_ctc at 132 SMs, vec2 (even K) row pitch = the least Kp > K with Kp = 2 mod 4, else the least
# odd Kp > K: par halves its gradient warps NW 8 -> 4 above Kp 160 and 4 -> 2 above Kp 320, and stops at Kp 800; pair
# needs Kp <= 533; the double-buffered warp kernel (every batch below 16 x SMs) Kp <= 1066.
K_LIMITS = [
    # (name, B, forced, K, expected kernel / NW, or None for CTCB_EINVAL)
    ("par-nw8", 1, "auto", 156, dict(kernel="par", warps=8, Kp=158)),
    ("par-nw4", 1, "auto", 158, dict(kernel="par", warps=4, Kp=162)),
    ("par-nw4-odd", 1, "auto", 159, dict(kernel="par", warps=4, Kp=161, vec2=0)),
    ("par-nw4-last", 1, "auto", 316, dict(kernel="par", warps=4, Kp=318)),
    ("par-nw2", 1, "auto", 318, dict(kernel="par", warps=2, Kp=322)),
    ("par-last", 1, "auto", 796, dict(kernel="par", warps=2, Kp=798)),
    ("par-to-warp", 1, "auto", 798, dict(kernel="warp", th=16, nbuf=2, Kp=802)),
    ("par-forced-too-wide", 1, "par", 798, None),
    ("pair-last", 133, "auto", 264, dict(kernel="pair", Kp=266)),
    ("pair-to-warp", 133, "auto", 266, dict(kernel="warp", th=16, nbuf=2, Kp=270)),
    ("pair-forced-last-even", 4, "pair", 528, dict(kernel="pair", Kp=530)),
    ("pair-forced-530", 4, "pair", 530, None),
    ("pair-forced-last", 4, "pair", 531, dict(kernel="pair", Kp=533, vec2=0)),
    ("pair-forced-532", 4, "pair", 532, None),
    ("warp-last", 1, "auto", 1064, dict(kernel="warp", Kp=1066)),
    ("warp-last-odd", 1, "auto", 1063, dict(kernel="warp", Kp=1065, vec2=0)),
    ("too-wide-1065", 1, "auto", 1065, None),
    ("too-wide-1066", 1, "auto", 1066, None),
]


@pytest.mark.parametrize("name,B,forced,K,expect", K_LIMITS, ids=[c[0] for c in K_LIMITS])
def test_k_limits(name, B, forced, K, expect, cuda, force):
    """At each limit the query and the call agree: the plan named runs and matches the oracle; beyond the last K any
    organisation can hold, and beyond a forced organisation's limit, the call returns CTCB_EINVAL."""
    T, L = 24, 6
    b = _make(B, T, K, L, seed=K + B, scale=1.0)
    if expect is None:
        force(forced)
        rc, plan = _plan(B, T, K, L)
        assert rc == -1 and plan is None
        r, _ = _run(cuda, b, check_rc=False)
        assert r == -1, r
        return
    _case(cuda, force, "klimit-" + name, b, expect, forced)


def test_forced_organisations_that_cannot_run_are_errors(cuda, force):
    """A forced organisation never quietly becomes another one."""
    from _ctcb import lib
    force("par")
    assert _plan(257, 10, 40, 10)[0] == -1 and b"256" in lib.ctcb_last_error()
    assert _plan(256, 10, 40, 10)[1]["kernel"] == "par"
    force("ckpt")
    assert _plan(8, 10, 40, 128)[0] == -1 and b"127" in lib.ctcb_last_error()
    assert _plan(8, 10, 40, 127)[1]["kernel"] == "ckpt"
    assert _plan(8, 10, 400, 20)[0] == -1
    for f in ("warp", "pair"):
        force(f)
        assert _plan(3000, 10, 40, 300)[1]["kernel"] == f


# ------------------------------------------------------------------------------------------------ blank position
@pytest.mark.parametrize("blank", ["zero", "last", "middle", "inside"])
@pytest.mark.parametrize("kern,forced,B", [("par", "auto", 4), ("pair", "auto", 140), ("ckpt", "ckpt", 8),
                                           ("warp", "warp", 8)])
def test_blank_position(kern, forced, B, blank, cuda, force):
    K, T, L = 37, 50, 20
    bl = {"zero": 0, "last": K - 1, "middle": K // 2, "inside": 5}[blank]
    b = _make(B, T, K, L, seed=bl + B, blank=bl)
    if blank == "inside":                   # a label equal to the blank index inside the sequence
        for s in b.seqs:
            s[len(s) // 2] = bl
            s[1] = bl
    _case(cuda, force, "blank-%s-%s" % (blank, kern), b, dict(kernel=kern), forced)


# ------------------------------------------------------------------------------------------------ trellis edges
def _trellis_batch(K=12, seed=5):
    """One utterance per edge, all in one batch."""
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


@pytest.mark.parametrize("P", [1, 2, 4])
@pytest.mark.parametrize("kern,forced", [("par", "auto"), ("pair", "pair"), ("ckpt", "ckpt"), ("warp", "warp")])
def test_trellis_edges(kern, forced, P, cuda, force):
    K = 12
    rows = _trellis_batch(K)
    Tmax = max(T for T, _ in rows)
    rng = np.random.RandomState(P)
    x = (rng.randn(len(rows), Tmax, K) * 1.5).astype(np.float32)
    b = Batch(x, [T for T, _ in rows], [s for _, s in rows])
    L = {1: 31, 2: 63, 4: 127}[P]                     # max_labels sets P
    res = _case(cuda, force, "trellis-%s-P%d" % (kern, P), b, dict(kernel=kern, P=P), forced, max_labels=L)
    skip = res[3]
    assert skip[5] == 1 and not skip[[4, 6, 7]].any() and np.isinf(res[1][8])


# ------------------------------------------------------------------------------------------------ batch edges
@pytest.mark.parametrize("kern,forced,B", [("par", "auto", 9), ("pair", "auto", 150), ("ckpt", "ckpt", 9),
                                           ("warp", "warp", 9)])
def test_batch_edges(kern, forced, B, cuda, force):
    """Ragged time-major batch (utt_stride = K, frame_stride = B K, the BRNN's layout); T_per_utt > Tmax is clamped,
    T_per_utt = 0 skips with an all-zero gradient; the same utterance at two positions gives the same bits."""
    K, T, L = 33, 70, 24
    b = _make(B, T, K, L, seed=B, layout="tb")
    b.lens[1] = T + 25                    # clamped to Tmax
    b.lens[2] = 0
    b.x[B - 1], b.lens[B - 1], b.seqs[B - 1] = b.x[0], b.lens[0], b.seqs[0]
    res = _case(cuda, force, "batch-%s" % kern, b, dict(kernel=kern), forced)
    plan, nll, g, skip, _ = res
    assert skip[2] == 1 and skip[1] == 0
    assert nll[0] == nll[B - 1] and np.array_equal(g[0], g[B - 1])


# ------------------------------------------------------------------------------------------------ zero mass
@pytest.mark.parametrize("kern,forced", [("par", "auto"), ("pair", "pair"), ("ckpt", "ckpt"), ("warp", "warp")])
def test_zero_mass(kern, forced, cuda, force):
    """Probability input with exact zeros: a required label's probability 0 on a frame where the alignment is forced
    (skip), and frames where every probability but one is 0 (one-hot rows)."""
    K, T = 10, 30
    rng = np.random.RandomState(3)
    p = rng.rand(4, T, K).astype(np.float64) + 0.05
    seqs = [np.array([1, 2, 3, 4, 5], np.int32)] * 4
    lens = [5, T, T, T]
    p[0, 2, 3] = 0.0                                   # T = |l|, distinct: label 3 must be emitted at frame 2
    p[2, 10:20] = 0.0
    p[2, 10:20, 0] = 1.0                               # blank only on ten frames
    p[3, 5, :] = 0.0
    p[3, 5, 4] = 1.0                                   # one frame that is label 4 only
    p /= p.sum(axis=2, keepdims=True)
    b = Batch(p.astype(np.float32), lens, seqs, is_prob=True)
    res = _case(cuda, force, "zero-mass-%s" % kern, b, dict(kernel=kern), forced)
    assert res[3][0] == 1 and not res[3][1:].any()


# ------------------------------------------------------------------------------------------------ range
def test_long_utterance_5000_frames(cuda, force):
    """A C4-length utterance: the float32 sum of log Z over 5000 frames and 300 labels (P = 16), logits and
    probabilities, on the default plan for one utterance.  The logits favour each label on a few frames of its own
    segment, as a trained net's do.  (With logits that carry no alignment at all, the gradient of one frame differed from
    the reference's; see DESIGN.md section 4.)"""
    T, K, L = 5000, 35, 300
    for is_prob in (False, True):
        b = _make(1, T, K, L, seed=11, ragged=False)
        seg = T // L
        for i, l in enumerate(b.seqs[0]):
            b.x[0, i * seg + seg // 2 - 2:i * seg + seg // 2 + 2, l] += 6.0
        if is_prob:
            b.x = _softmax64(b.x.reshape(T, K)).reshape(1, T, K).astype(np.float32)
            b.is_prob = True
        _case(cuda, force, "long-5000-%s" % ("prob" if is_prob else "logit"), b, dict(kernel="par", P=16))


@pytest.mark.parametrize("kern,forced", [("par", "auto"), ("ckpt", "ckpt"), ("warp", "warp")])
def test_emission_below_float32_normal_range(kern, forced, cuda, force):
    """A label whose logit is 90 nats below its frame's maximum on a frame where the alignment is forced (T = |l|,
    distinct labels): its probability, e^-90 / Z ~ 1e-39, is a float32 subnormal.  Given as probabilities the kernel keeps
    it and matches the oracle.  Given as logits the fused softmax computes it with ex2.approx.ftz, which flushes it to
    0: the only path dies and the kernel skips the utterance where the reference, fed the float32 softmax, returns a
    finite loss.  That is the kernel's documented behaviour (DESIGN.md section 4); this test pins it."""
    K, L = 16, 8
    rng = np.random.RandomState(9)
    seq = (1 + rng.permutation(K - 1)[:L]).astype(np.int32)
    x = rng.randn(2, L, K).astype(np.float32)
    x[:, 3, :] = 0.0
    x[:, 3, 0] = 45.0
    x[:, 3, seq[3]] = -45.0                            # 90 nats below the frame's maximum
    p32 = _softmax64(x.reshape(2 * L, K)).reshape(2, L, K).astype(np.float32)
    assert 0.0 < p32[0, 3, seq[3]] < np.finfo(np.float32).tiny
    t0 = time.time()
    force(forced)
    bp = Batch(p32, [L, L], [seq, seq], is_prob=True)
    res = _run(cuda, bp, plan_expect=dict(kernel=kern), what="subnormal-prob")
    gerr, nerr, n = _compare(bp, res)
    _report("subnormal-prob-%s" % kern, res[0], gerr, nerr, n, t0, forced=forced)
    assert n["ok"] == 2
    bl = Batch(x, [L, L], [seq, seq])
    plan, nll, g, skip, _ = _run(cuda, bl, plan_expect=dict(kernel=kern), what="subnormal-logit")
    o_nll, _, o_skip = ctc_oracle.ctc_loss(np.asfortranarray(p32[0].T.astype(np.float64)), seq)
    assert not o_skip and np.isfinite(o_nll)
    assert (skip == 1).all() and not g.any(), (skip, nll)


# ------------------------------------------------------------------------------------------------ identity
def test_identity_across_organisations(cuda, force):
    """The same inputs on every organisation.  Probability input: every organisation gives the same bits.  Logits: the
    fused softmax sums a row's normaliser over 2 lanes with 16-frame tiles (par, pair, warp 16) and over 4 lanes with
    8-frame tiles (ckpt, warp 8), so Z, the gradient and log Z are the same bits within each tile height and differ in
    the last bits across the two."""
    K, T, L = 40, 60, 25
    B = 16 * H100_SMS + 20
    base = _make(B, T, K, L, seed=77)
    out = {}
    for is_prob in (False, True):
        x = base.x if not is_prob else _softmax64(base.x.reshape(-1, K)).reshape(base.x.shape).astype(np.float32)
        big = Batch(x, base.lens, base.seqs, is_prob=is_prob)
        small = Batch(x[:200], base.lens[:200], base.seqs[:200], is_prob=is_prob)
        runs = {}
        for name, batch, forced, expect in (("par", small, "par", dict(kernel="par", th=16)),
                                            ("pair", small, "pair", dict(kernel="pair", th=16)),
                                            ("warp16", small, "warp", dict(kernel="warp", th=16, nbuf=2)),
                                            ("ckpt", small, "ckpt", dict(kernel="ckpt", th=8)),
                                            ("ckpt-big", big, "ckpt", dict(kernel="ckpt", th=8)),
                                            ("warp8-big", big, "warp", dict(kernel="warp", th=8, nbuf=1)),
                                            ("pair-big", big, "pair", dict(kernel="pair", th=16))):
            force(forced)
            plan, nll, g, skip, _ = _run(cuda, batch, plan_expect=expect, what=name)
            runs[name] = (nll[:200], g[:200], skip[:200])
        gerr, nerr, n = _compare(small, (None, runs["par"][0], runs["par"][1], runs["par"][2], np.array([SENTINEL])))
        same = lambda a, b: all(np.array_equal(u, v) for u, v in zip(runs[a], runs[b]))
        tiles16, tiles8 = ("par", "pair", "warp16", "pair-big"), ("ckpt", "ckpt-big", "warp8-big")
        for grp in (tiles16, tiles8):
            for o in grp[1:]:
                assert same(grp[0], o), (is_prob, grp[0], o)
        d_g = float(np.abs(runs["par"][1] - runs["ckpt"][1]).max())
        d_nll = float(np.max(np.abs(runs["par"][0] - runs["ckpt"][0]) / np.abs(runs["par"][0])))
        ulp_g = d_g / np.finfo(np.float32).eps
        out["prob" if is_prob else "logit"] = dict(grad_diff_8_vs_16=d_g, nll_rel_diff_8_vs_16=d_nll,
                                                  grad_err=gerr, nll_err=nerr)
        if is_prob:
            assert same("par", "ckpt"), "probability input differs between tile heights"
        else:
            assert d_g <= 8 * np.finfo(np.float32).eps and d_nll <= 8 * np.finfo(np.float32).eps, (d_g, d_nll, ulp_g)
        assert gerr <= BOUNDS["par"][0] and nerr <= BOUNDS["par"][1]
    print(json.dumps(dict(ctc="identity", **out)))


# ------------------------------------------------------------------------------------------------ workspace
def test_brnn_smaller_call_than_maxB_fits_its_ctc_workspace(cuda):
    """A net sized for maxB = 260 (the C3-like widths of the two-CTA-cluster config) takes a training call of 200
    utterances at Tmax = maxT: the frame-parallel CTC kernel then spills two planes per utterance, more than one plane
    for each of 260, and the CTC area sized for maxB must hold them."""
    import nnets.brnnet as brnnet
    import recipes
    from oracle import brnn_oracle
    D, K, H, N, tl, T, L, maxB, B = 41, 32, 1024, 3, 2, 16, 5, 260, 200
    datas, labelss = recipes.synth_batch(D, K, [T] * B, [L] * B, seed=34)
    np.random.seed(33)
    nn = brnnet.NNet(D, K, H, N, T, temporalLayer=tl, maxUtts=maxB, maxLabels=L)
    nn.initParams()
    costs, _, skips = nn.costAndGradBatch(datas, labelss)
    del nn
    np.random.seed(33)
    on = brnn_oracle.NNet(D, K, H, N, T, temporalLayer=tl, dtype=np.float64)
    on.initParams()
    o_costs = np.array([ctc_oracle.ctc_loss(np.asfortranarray(on.forward(d)[3].astype(np.float64)), l)[0]
                        for d, l in zip(datas, labelss)])
    err = float(np.max(np.abs(costs - o_costs) / np.abs(o_costs)))
    print(json.dumps(dict(ctc="brnn-maxB260-B200", cost_rel_err=err)))
    assert not skips.any() and np.isfinite(costs).all()
    assert err <= 1e-4, err
