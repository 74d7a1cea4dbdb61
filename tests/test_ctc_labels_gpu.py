"""Malformed label sequences in the CTC kernel (ctcb_ctc_loss_grad_f32) on every plan, and in the training step.

Utterance u is malformed when its label count label_off[u+1] - label_off[u] is negative or above max_labels, or one of
its labels lies outside [0, K) (include/ctcb200.h).  The kernel checks that on the device before it reads a row and
skips the utterance exactly as one with T_per_utt = 0.  Each case below mixes malformed utterances into a batch of good
ones and runs three launches of the same shape (same B, so the same plan, checked with ctcb_debug_ctc_plan first):

  * bad:  the malformed sequences;
  * good: each malformed sequence replaced by a valid one of the same length (at most max_labels);
  * zero: the good sequences, with T_per_utt = 0 for the utterances that are malformed in `bad`.

Every malformed utterance of `bad` gives the nll, skip and gradient bytes of `zero`, every other utterance those of
`good`, and nothing outside the batch's elements is written (guard bands before and after the gradient, its gap columns,
guards around nll and skip).  Utterance 0 is a maximal valid sequence (max_labels labels, among them 0 and K - 1),
computed, not skipped, and held to oracle.ctc_oracle under test_ctc_plans_gpu.BOUNDS.

The labels reach: K, K + 1, K + Kp (the next row of a shared tile), 2^30, INT_MAX, -1 and INT_MIN; in the first
position, a middle one, the last one and the last pair of a lane; on utterances of 1 frame (the short-utterance loss),
2 .. |l| - 1 frames, Tmax frames and 0 frames.  The counts: max_labels + 1, the lanes' capacity 32P - 1 and 32P where
max_labels is below it, 32P + 40, and a label_off that decreases."""
import ctypes
import json
import time

import numpy as np
import pytest

import recipes
from oracle import ctc_oracle
from recipes import Batch, knobs  # noqa: F401  (knobs: fixture of force)
from test_ctc_plans_gpu import BOUNDS, H100_SMS, SENTINEL, _check_plan, _compare, _plan, force  # noqa: F401

pytestmark = pytest.mark.gpu
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
GUARD = 64                      # floats of guard band on either side of the gradient (keeps the 256-byte alignment)
NLL_GUARD, SKIP_GUARD = -3.5, -7
REACHED = set()                 # (organisation, P) of the cases run
LABEL_KINDS = ("K", "K+1", "K+Kp", "2^30", "INT_MAX", "-1", "INT_MIN")
POSITIONS = ("first", "middle", "last", "lane-last")
FRAMES = ("1", "short", "Tmax", "0")


def _label_value(kind, K, Kp):
    return {"K": K, "K+1": K + 1, "K+Kp": K + Kp, "2^30": 2 ** 30, "INT_MAX": INT_MAX, "-1": -1,
            "INT_MIN": INT_MIN}[kind]


def _position(kind, n, P):
    if kind == "first":
        return 0
    if kind == "middle":
        return n // 2
    if kind == "last":
        return n - 1
    return max(i for i in range(n) if i % P == P - 1) if n >= P else n - 1     # the last pair of a lane


def _frames(kind, n, Tmax):
    return {"1": 1, "short": max(2, n // 2), "Tmax": Tmax, "0": 0}[kind]


# ------------------------------------------------------------------------------------------------ one launch
def _launch(torch, b, seqs, lens, max_labels, off=None):
    """ctcb_ctc_loss_grad_f32 on the activations of b with the given label sequences and frame counts (off: label_off,
    default their prefix sums).  Returns (nll bytes [B], skip [B], gradient [B][Tmax][K] bytes, what lies outside)."""
    import _ctcb
    from _ctcb import lib, check, ptr
    B = b.B
    x = np.concatenate([np.full(GUARD, np.nan, np.float32), b.flat(np.nan), np.full(GUARD, np.nan, np.float32)])
    d_x = torch.from_numpy(x).cuda()
    d_g = torch.from_numpy(np.full(b.n + 2 + 2 * GUARD, SENTINEL, dtype=np.float32)).cuda()
    lab = np.concatenate([np.asarray(s, np.int64) for s in seqs] + [np.zeros(1, np.int64)]).astype(np.int32)
    if off is None:
        off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
    d_lab = torch.from_numpy(lab).cuda()
    d_off = torch.from_numpy(np.asarray(off, np.int32)).cuda()
    d_len = torch.tensor(lens, dtype=torch.int32).cuda()
    nll = torch.full((B + 2 * GUARD,), NLL_GUARD, device="cuda")
    skip = torch.full((B + 2 * GUARD,), SKIP_GUARD, dtype=torch.int32, device="cuda")
    nws = int(lib.ctcb_ctc_workspace_bytes(B, b.Tmax, max_labels))
    ws = torch.empty(max(nws, 8), dtype=torch.uint8, device="cuda")
    check(lib.ctcb_ctc_loss_grad_f32(d_x.data_ptr() + 4 * GUARD, int(b.is_prob), b.us, b.fs, ptr(d_lab), ptr(d_off),
                                     ptr(d_len), B, b.Tmax, b.K, max_labels, b.blank, d_g.data_ptr() + 4 * GUARD,
                                     nll.data_ptr() + 4 * GUARD, skip.data_ptr() + 4 * GUARD, ptr(ws), nws,
                                     _ctcb.current_stream()))
    torch.cuda.synchronize()
    g = d_g.cpu().numpy()
    inside = np.zeros(g.shape, bool)
    inside[GUARD + b.idx] = True
    nll, skip = nll.cpu().numpy(), skip.cpu().numpy()
    outside = dict(grad=g[~inside], nll=np.concatenate([nll[:GUARD], nll[GUARD + B:]]),
                   skip=np.concatenate([skip[:GUARD], skip[GUARD + B:]]))
    return nll[GUARD:GUARD + B].view(np.uint32), skip[GUARD:GUARD + B], g[GUARD + b.idx].view(np.uint32), outside


# ------------------------------------------------------------------------------------------------ one case
def _malformed_case(torch, force, name, kern, forced, B, P, max_labels, K=40, layout=("bt", 0), is_prob=False,
                    expect=None, shift=0):
    t0 = time.time()
    force(forced)
    Tmax = max_labels + max_labels // 4 + 8
    rng = np.random.RandomState(1000 * P + B + shift)
    b = recipes.ctc_batch(B, Tmax, K, max_labels, seed=7 * P + B + shift, is_prob=is_prob, layout=layout[0],
                          fs_pad=layout[1])
    # utterance 0: a maximal valid sequence with the edge labels, on all Tmax frames
    s0 = recipes.ctc_labels(rng, max_labels, K, b.blank)
    s0[0], s0[max_labels // 2], s0[-1] = K - 1, 0, K - 1
    b.seqs[0], b.lens[0] = s0, Tmax
    rc, plan = _plan(B, Tmax, K, max_labels, 256, 256, b.us, b.fs)
    assert rc == 0, plan
    _check_plan(plan, dict(expect or {}, kernel=kern, P=P), torch, name)
    Kp = plan["Kp"]
    REACHED.add((kern, P))
    cap = 32 * P - 1
    counts = sorted({max_labels + 1, cap, cap + 1, cap + 41} - set(range(max_labels + 1)))

    # the malformed utterances: two of every three, the last one with a decreasing label_off
    good, bad, lens, kinds = list(b.seqs), list(b.seqs), list(b.lens), {}
    k = shift
    for u in range(1, B):
        if u % 3 == 0 and u != B - 1:
            continue
        fr = FRAMES[(k // len(POSITIONS)) % len(FRAMES)]
        if u == B - 1:
            kinds[u] = ("decreasing-label_off", fr)
        elif k % 5 == 4:
            n = counts[(k // 5) % len(counts)]
            s = recipes.ctc_labels(rng, n, K, b.blank)
            if n > cap:
                s[cap] = K                                   # the pair no lane holds
            bad[u], good[u] = s, s[:max_labels]
            kinds[u] = ("count", n, fr)
        else:
            s = np.array(b.seqs[u], np.int64)
            if len(s) < 3:
                s = recipes.ctc_labels(rng, 3, K, b.blank).astype(np.int64)
                good[u] = s.astype(np.int32)
            kind, pos = LABEL_KINDS[k % len(LABEL_KINDS)], POSITIONS[k % len(POSITIONS)]
            i = _position(pos, len(s), P)
            s = s.copy()
            s[i] = _label_value(kind, K, Kp)
            bad[u] = s
            kinds[u] = (kind, pos, i, fr)
        lens[u] = _frames(fr, len(good[u]), Tmax)
        k += 1
    off_bad = np.concatenate([[0], np.cumsum([len(s) for s in bad])])
    off_bad[B] = off_bad[B - 1] - 5                          # utterance B - 1: label count -5
    zero = [0 if u in kinds else t for u, t in enumerate(lens)]

    r_bad = _launch(torch, b, bad, lens, max_labels, off_bad)
    r_good = _launch(torch, b, good, lens, max_labels)
    r_zero = _launch(torch, b, good, zero, max_labels)
    for r in (r_bad, r_good, r_zero):
        out = r[3]
        assert (out["grad"] == SENTINEL).all(), "a guard band or gap column of the gradient was written"
        assert (out["nll"] == NLL_GUARD).all() and (out["skip"] == SKIP_GUARD).all(), "an nll or skip guard was written"
    nll, skip, g = r_bad[:3]
    for u in range(B):
        ref = r_zero if u in kinds else r_good
        assert nll[u] == ref[0][u] and skip[u] == ref[1][u], (name, u, kinds.get(u), nll[u], ref[0][u], skip[u])
        assert np.array_equal(g[u], ref[2][u]), (name, u, kinds.get(u))
        if u in kinds:
            assert skip[u] == 1 and not g[u].any(), (name, u, kinds[u])
    assert skip[0] == 0 and np.isfinite(nll[:1].view(np.float32)).all(), "the maximal valid sequence was skipped"

    # utterance 0 against the oracle
    b.lens = lens
    b.seqs = good
    res = (plan, nll.view(np.float32).astype(np.float64), g.view(np.float32).astype(np.float64), skip,
           np.array([SENTINEL]))
    gerr, nerr, n = _compare(b, res, utts=[0])
    gb, nb = BOUNDS[kern]
    print(json.dumps(dict(ctc_labels=name, plan=plan, forced=forced, B=B, max_labels=max_labels, K=K, layout=layout,
                          is_prob=is_prob, malformed=len(kinds), kinds=sorted(set(str(v[0]) for v in kinds.values())),
                          grad_err=gerr, nll_err=nerr, grad_bound=gb, nll_bound=nb, seconds=round(time.time() - t0, 2))))
    assert n["ok"] == 1, n
    assert gerr <= gb and nerr <= nb, (name, gerr, nerr)
    return kinds


# ------------------------------------------------------------------------------------------------ cases
LAYOUTS = (("bt", 0), ("tb", 0), ("bt", 2), ("tb", 3))     # utterance-major, the step's time-major, padded frames


def _cases():
    cases = []
    labels = {1: (31, 16), 2: (63, 32), 4: (127, 64), 8: (255, 128), 16: (511, 256)}
    for P, mls in labels.items():
        for kern, forced, B in (("par", "auto", 24), ("par", "par", 24), ("pair", "auto", 140), ("pair", "pair", 24),
                                ("warp", "warp", 24), ("ckpt", "ckpt", 24)):
            if kern == "ckpt" and P > 4:
                continue
            for ml in mls:
                cases.append((kern, forced, B, P, ml, None))
    # ckpt chosen automatically (more utterances than the pair kernel's wave, K <= 64 P); the warp kernel's one-buffer
    # tiles (B >= 16 x SMs): 16 frames, and 8 frames at P <= 2, automatic and forced
    cases += [("ckpt", "auto", 1100, 1, 31, None), ("ckpt", "auto", 1100, 4, 100, None),
              ("warp", "warp", 2200, 4, 127, dict(th=16, nbuf=1)), ("warp", "auto", 2200, 8, 140, dict(th=16, nbuf=1)),
              ("warp", "warp", 2200, 2, 63, dict(th=8, nbuf=1)), ("warp", "auto", 2200, 1, 31, dict(th=8, nbuf=1)),
              ("warp", "warp", 24, 2, 40, dict(th=16, nbuf=2))]
    out = []
    for i, (kern, forced, B, P, ml, expect) in enumerate(cases):
        K = 80 if (kern, forced, P) == ("warp", "auto", 1) else 40         # K > 64 P: the spill, not the checkpoints
        lay = LAYOUTS[i % len(LAYOUTS)]
        is_prob = i % 3 == 1
        out.append(pytest.param(kern, forced, B, P, ml, K, lay, is_prob, expect, i,
                                id="%s-%s-B%d-P%d-L%d-%s%d-%s" % (kern, forced, B, P, ml, lay[0], lay[1],
                                                                 "prob" if is_prob else "logit")))
    return out


@pytest.mark.parametrize("kern,forced,B,P,max_labels,K,layout,is_prob,expect,shift", _cases())
def test_malformed_utterances_skip_without_touching_the_batch(kern, forced, B, P, max_labels, K, layout, is_prob,
                                                             expect, shift, cuda, force):
    _malformed_case(cuda, force, "labels-%s-%s-P%d-L%d" % (kern, forced, P, max_labels), kern, forced, B, P,
                    max_labels, K=K, layout=layout, is_prob=is_prob, expect=expect, shift=shift)


# ------------------------------------------------------------------------------------------------ the training step
STEP_NETS = {"bi_relu": dict(H=64, N=3, K=29, kw=dict(temporalLayer=2)),
             "lstm_bi": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm"))}
D_IN, MAXT, MAXB, MAXL = 23, 40, 7, 6


def _step_net(c):
    import nnets.brnnet as brnnet
    np.random.seed(17)
    nn = brnnet.NNet(D_IN, c["K"], c["H"], c["N"], MAXT, maxUtts=MAXB, maxLabels=MAXL, **c["kw"])
    nn.initParams()
    return nn


def _delta(nn, j, T, B):
    from _ctcb import lib
    off, width = ctypes.c_size_t(), ctypes.c_int32()
    if lib.ctcb_brnn_activation_offset(ctypes.byref(nn._cfg), 7, j, ctypes.byref(off), ctypes.byref(width)):
        return None
    return nn._ws[off.value:off.value + 4 * T * B * width.value].view(nn._torch.float32).view(T, B, width.value)


@pytest.mark.parametrize("bad", ["K", "-1", "INT_MAX"])
@pytest.mark.parametrize("name", list(STEP_NETS))
def test_step_skips_a_malformed_utterance(name, bad, cuda):
    """ctcb_brnn_cost_and_grad with valid labels packed and then one utterance's labels overwritten on the device: that
    utterance is skipped, the statistics tail leaves its cost out, its rows of every map's delta are 0 (+0.0 in the ReLU
    net), and the other utterances' rows of the top delta keep their bits."""
    torch = cuda
    c = STEP_NETS[name]
    K = c["K"]
    nn = _step_net(c)
    rng = np.random.RandomState(3)
    lens = [int(t) for t in rng.randint(12, MAXT + 1, size=MAXB)]
    datas, labelss = recipes.synth_batch(D_IN, K, lens, [int(x) for x in rng.randint(2, MAXL + 1, size=MAXB)], seed=5)
    m = 2
    value = {"K": K, "-1": -1, "INT_MAX": INT_MAX}[bad]
    runs = {}
    for what in ("good", "bad"):
        batch = nn.swap_batches().pack(datas, labelss).upload()
        if what == "bad":
            o = int(batch.h_off[m]) + len(labelss[m]) // 2
            batch.d_labels[o] = value
        cost, skip = nn.costAndGradDevice(batch)
        torch.cuda.synchronize()
        T, B = batch.Tmax, batch.B
        deltas = {j: _delta(nn, j, T, B) for j in range(1, nn.numLayers + 2)}
        runs[what] = dict(cost=cost.cpu().numpy().copy(), skip=skip.cpu().numpy().copy(),
                          stats=nn.stats.cpu().numpy().astype(np.float64),
                          deltas={j: d.cpu().numpy().copy() for j, d in deltas.items() if d is not None})
    good, bad = runs["good"], runs["bad"]
    assert not good["skip"].any(), good["skip"]
    assert bad["skip"][m] == 1 and not np.delete(bad["skip"], m).any(), bad["skip"]
    ok = bad["skip"] == 0
    assert np.array_equal(bad["cost"][ok].view(np.uint32), good["cost"][ok].view(np.uint32))
    st = bad["stats"]
    want = bad["cost"][ok].astype(np.float64)
    assert st[0] == MAXB - 1 and st[2] == 1 and st[3] == 0, st
    assert abs(st[1] - want.sum()) <= MAXB * 2.0 ** -23 * np.abs(want).sum(), (st, want.sum())
    for j, d in bad["deltas"].items():
        # the LSTM's BPTT carries the zero gradient through its gate derivatives as +-0.0, as for any utterance the CTC
        # skips; the ReLU step's deltas are +0.0 bits
        if c["kw"].get("cell") == "lstm":
            assert (d[:, m] == 0.0).all(), "map %d: the malformed utterance's delta is not 0" % j
        else:
            assert not d[:, m].view(np.uint32).any(), "map %d: the malformed utterance's delta is not +0.0" % j
    top = nn.numLayers + 1
    others = [u for u in range(MAXB) if u != m]
    assert np.array_equal(bad["deltas"][top][:, others].view(np.uint32), good["deltas"][top][:, others].view(np.uint32))
    print(json.dumps({"step_malformed_%s_%s" % (name, bad): dict(maps=sorted(bad["deltas"]), stats=st.tolist())}))


@pytest.mark.parametrize("rule", ["nesterov", "adam"])
def test_step_of_malformed_utterances_only_changes_nothing(rule, cuda):
    """Every utterance of the step malformed: n_valid = 0, so one SGD step leaves w and the optimiser's states bit for
    bit (Nesterov's look-ahead with zero velocity is undone exactly), and the step counter advances once."""
    import sgd
    torch = cuda
    c = STEP_NETS["bi_relu"]
    nn = _step_net(c)
    opt = sgd.SGD(nn, MAXT, alpha=1e-3, optimizer=rule, momentum=0.9, maxGradNorm=5.0, batchSize=MAXB, verbose=False)
    rng = np.random.RandomState(4)
    lens = [int(t) for t in rng.randint(12, MAXT + 1, size=4)]
    datas, labelss = recipes.synth_batch(D_IN, c["K"], lens, [3] * 4, seed=6)
    batch = nn._batch.pack(datas, labelss).upload()
    batch.d_labels[:12] = c["K"]
    w0 = nn.params.cpu().numpy().copy()
    s0 = [opt._flat[n].cpu().numpy().copy() for n in sgd.OPTIMIZERS[rule]]
    opt.it += 1
    opt.step_device(batch, opt._momentum_now())
    torch.cuda.synchronize()
    st = nn.stats.cpu().numpy()
    assert st[0] == 0 and st[2] == 4, st
    assert np.array_equal(nn.params.cpu().numpy().view(np.uint32), w0.view(np.uint32))
    for n, s in zip(sgd.OPTIMIZERS[rule], s0):
        assert np.array_equal(opt._flat[n].cpu().numpy().view(np.uint32), s.view(np.uint32)), n
    if opt._step is not None:
        assert int(opt._step.item()) == opt.it == 1


def test_every_organisation_and_pairs_per_lane_was_reached(cuda):
    """The malformed-label cases above ran on every organisation at every P it supports."""
    want = {(k, P) for k in ("par", "pair", "warp") for P in (1, 2, 4, 8, 16)} | {("ckpt", P) for P in (1, 2, 4)}
    missing = sorted(want - REACHED)
    if missing and cuda.cuda.get_device_properties(0).multi_processor_count != H100_SMS:
        pytest.skip("plans not reachable on this device: %s" % missing)
    assert not missing, missing
