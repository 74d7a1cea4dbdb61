"""GPU unit test of the clipped-ReLU recurrent sweep on its own (ctcb_brnn_sweep_f32) on every plan its planner can
choose, against float64 steps of brnnet.py:144-152 (forward) and :208-224 (BPTT) taken from the GPU's own states.

The planner (select_sweep, csrc/sweep.cu) picks one of three kernels: the tensor-core kernel sweep_tc_kernel<NP>
(H >= 1024), the cluster kernel sweep_cluster_kernel<KI, NB> (H = 128/256/512 while one wave of clusters holds the
batch) and the generic cooperative kernel sweep_kernel<KI> (everything else; KI = H / 32 at H = 128, 256, 512, 1024,
else 0).  Every case names the plan it targets and checks it with ctcb_debug_sweep_plan before launching; for the
generic kernel that includes its CTAs per SM, against the table below.  CTCB_SWEEP=reread and CTCB_SWEEP_PARTS steer
the generic kernel, the other CTCB_SWEEP* knobs the others; tests set them in process (recipes.knobs).

Forward, element-wise and step-local: each output x_t against x64 = clip(pre_t + W h_{t-1}, 0, maxAct) in float64, with
h_{t-1} the GPU's own state of the step before, |x - x64| <= C u S, u = 2^-24, S = |pre_t| + |W| |h_{t-1}|, no floor.
Where x64 is clipped by more than the bound, x is exactly 0 or maxAct; where h_{t-1} is all zero (each direction's first
frame, and the frame after one that drives every state below 0), x is exactly clip(pre_t).  BPTT the same on
dF_t = mask_t (d_t + W^T dF_{t+1}), mask_t = 0 < act_t < maxAct of the states the BPTT is given, S = |d_t| +
|W^T| |dF_{t+1}|; masked elements are exactly +0.0.  The step-local bound does not grow with T: C is one constant per
kernel family, and for the tensor-core kernel c0 + c1 L, L = k-blocks per K-slice (H / CS / 32).  A TF32 emulation of
the same step (both operands truncated to 10 mantissa bits as the kernel truncates them, only the hi.hi product, in
float64) must err by at least TF32_MARGIN times the bound in every case with T >= 2.

Exact, in every case: outputs start as NaN and padded frames come back +0.0; NaN guard bands around pre, W, the outputs,
the incoming deltas and the masks' states are unchanged, and so are the bytes behind ctcb_brnn_sweep_workspace_bytes in
the scratch; the error words are 0; a rerun gives the same bytes; d 2^-20 gives dF 2^-20 where nothing comes near the
subnormals.  And the bits do not depend on the plan: every NB of the cluster kernel, every partition count and KI versus
the re-read path of the generic kernel, any number of utterance splits (and any wgmma N) of the tensor-core kernel, and
each direction of a bi-directional launch equals a uni-directional launch of its own.  Each case prints its plan and
ratios as one JSON line (pytest -s)."""
import ctypes
import json
import time

import numpy as np
import pytest

from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
MAXACT = 20.0
KERNELS = ("generic", "cluster", "tensor-core")
TC, CL, GEN = KERNELS[2], KERNELS[1], KERNELS[0]
H100_SMS = 132             # the plans below are laid out for the 132-SM H100 SXM; other parts skip a plan they cannot reach
# Bounds on |x - x64| / (u S), at most 4x the largest ratio measured on an H100 80GB HBM3 (700 W) over the cases of this
# file, forward and BPTT (DESIGN.md section 3): generic 1.79, cluster 2.02; tensor-core 7.5 at L = 4, 13.0 at L = 8,
# 29.9 at L = 16 (H = 1024 on clusters of 2, the tightest: bound 3.75x), 40.3 at L = 32, 50.7 at L = 40.  The TF32
# emulation measured at least 10.5x the bound (tensor-core, L = 32), 196x (generic) and 419x (cluster).
C_FFMA = {GEN: 7.0, CL: 8.0}
TC_C0, TC_C1 = 16.0, 6.0
TF32_MARGIN = 8.0
TINY = 2.0 ** -60          # d 2^-20 and its products with weights stay normal above this
SCALE = np.float32(2.0 ** -20)
GUARD = 64                 # NaN floats on each side of every buffer; 256 bytes keep the buffers' 16-byte alignment
NAN_BITS = np.float32(np.nan).view(np.uint32)
# CTAs of 256 threads per SM of sweep_kernel<KI> by registers (ptxas: KI=0 80, KI=4 and 8 96, KI=16 126, KI=32 206);
# shared memory (8 (ceil4(H) + 4) floats + 1 KB per CTA of the SM's 228 KB) may allow fewer.
REG_PER_SM = {0: 3, 4: 2, 8: 2, 16: 2, 32: 1}
SM_SMEM, CTA_RESERVED = 228 * 1024, 1024
GEN_REG_H = (128, 256, 512, 1024)


def _bound(plan, H):
    if plan["kernel"] == TC:
        return TC_C0 + TC_C1 * (H // plan["CS"] // 32)
    return C_FFMA[plan["kernel"]]


# ------------------------------------------------------------------------------------------------ plans
def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _smem(H):
    return 8 * ((H + 3) // 4 * 4 + 4) * 4


def _expect_generic(H, B, ndir, sms, reread=False, parts=None):
    """The generic kernel's plan select_sweep makes on a device of `sms` SMs, or None where it refuses."""
    ki = H // 32 if H in GEN_REG_H and not reread else 0
    if _smem(H) > 227 * 1024:
        return None
    per_sm = min(REG_PER_SM[ki], SM_SMEM // (_smem(H) + CTA_RESERVED))
    slices = -(-H // 32)
    cap = per_sm * sms
    if ndir * slices > cap:
        return None
    p = cap // (ndir * slices)
    if parts:
        if parts > p:
            return None
        p = parts
    return dict(kernel=GEN, KI=ki, parts=max(1, min(p, -(-B // 8), 500)), per_sm=per_sm)


def _plan_rc(H, B, ndir):
    """(rc, plan) of ctcb_debug_sweep_plan under the knobs in effect."""
    from _ctcb import lib
    out = (ctypes.c_int32 * 8)()
    rc = lib.ctcb_debug_sweep_plan(H, B, ndir, out)
    if rc != 0:
        return rc, None
    k = out[0]
    plan = dict(kernel=KERNELS[k], KI=out[1], CS=out[2])
    plan[("parts", "NB", "NS")[k]] = out[3]
    if k == 0:
        plan["per_sm"] = out[7]
    if k == 2:
        plan.update(NP=out[4], stages=out[5], partial_own=out[6])
    return rc, plan


def _plan(H, B, ndir):
    rc, plan = _plan_rc(H, B, ndir)
    from _ctcb import lib
    assert rc == 0, lib.ctcb_last_error()
    return plan


def _check_plan(H, B, ndir, expect, torch):
    plan = _plan(H, B, ndir)
    wrong = {k: (v, plan.get(k)) for k, v in expect.items() if plan.get(k) != v}
    if wrong:
        msg = "H=%d B=%d ndir=%d: planned %s, this case targets %s" % (H, B, ndir, plan, expect)
        if _sms(torch) != H100_SMS:
            pytest.skip("plan not reachable on this device: " + msg)
        pytest.fail(msg)
    if plan["kernel"] == GEN:        # the generic plan in full, from the register table and this device's SM count
        want = _expect_generic(H, B, ndir, _sms(torch), _KNOBS.get("CTCB_SWEEP") == "reread", _knob_parts())
        assert plan == dict(want, CS=0), (plan, want)
    return plan


# the generic knobs in effect, as the tests set them (recipes.knobs restores them)
_KNOBS = {}


def _set_knob(knobs, name, value):
    knobs(name, value)
    _KNOBS[name] = value


def _knob_parts():
    v = _KNOBS.get("CTCB_SWEEP_PARTS", "auto")
    return None if v == "auto" else int(v)


@pytest.fixture
def gknobs(knobs):
    """knobs that also remembers CTCB_SWEEP and CTCB_SWEEP_PARTS for _check_plan's generic expectation."""
    _KNOBS.clear()
    yield lambda name, value: _set_knob(knobs, name, value)
    _KNOBS.clear()


def _natural_family(H):
    """The kernel family the planner picks for a layer size at a small batch, under the knobs in effect."""
    return _plan(H, 1, 2)["kernel"]


# what the cases ran
SEEN = dict(gen=set(), cl=set(), np=set(), own=set(), cs=set(), coop=set(), empty=0, multi16=0, cases=0)


def _note(plan, B):
    if plan["kernel"] == GEN:
        SEEN["gen"].add(plan["KI"])
        ntiles = -(-B // 8)
        tpp = -(-ntiles // plan["parts"])
        if tpp * (plan["parts"] - 1) >= ntiles:
            SEEN["empty"] += 1
        last = (ntiles - 1) // tpp
        if B % 8 and min(ntiles, (last + 1) * tpp) - last * tpp >= 16:
            SEEN["multi16"] += 1
    elif plan["kernel"] == CL:
        SEEN["cl"].add((plan["KI"], plan["NB"]))
    else:
        SEEN["np"].add(plan["NP"])
        SEEN["own"].add(plan["partial_own"])
        SEEN["cs"].add(plan["CS"])
        SEEN["coop"].add(_KNOBS.get("CTCB_SWEEP_TC_COOP", "1"))


# ------------------------------------------------------------------------------------------------ one sweep
def _buf(torch, a):
    """A device copy of float32 array a inside NaN guard bands: (whole buffer, view of a)."""
    whole = torch.full((a.size + 2 * GUARD,), float("nan"), device="cuda")
    whole[GUARD:GUARD + a.size] = torch.from_numpy(np.ascontiguousarray(a, np.float32).ravel()).cuda()
    return whole, whole[GUARD:GUARD + a.size].view(a.shape)


def _guards_intact(whole):
    bits = whole.cpu().numpy().view(np.uint32)
    return bool((bits[:GUARD] == NAN_BITS).all() and (bits[-GUARD:] == NAN_BITS).all())


def _same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32),
                                                 np.ascontiguousarray(b).view(np.uint32))


class Sweep:
    """One sweep problem: lengths, pre-activations [T][B][H], recurrent matrices (one per direction), incoming deltas,
    and the states whose masks the BPTT takes (None: the GPU's own forward states; "edges": those with some entries
    replaced by the mask's boundary values)."""

    def __init__(self, torch, lens, pre, Ws, d, act="own"):
        self.torch, self.lens = torch, np.asarray(lens, np.int32)
        self.T, self.B, self.H = pre.shape
        self.ndir = len(Ws)
        self.pre, self.Ws, self.d, self.act = pre, Ws, d, act

    def run(self, d=None, fwd=None):
        """Forward then BPTT on fresh buffers (fwd: a previous run whose forward states and masks the BPTT reads)."""
        from _ctcb import lib, check
        torch, T, B, H, nd = self.torch, self.T, self.B, self.H, self.ndir
        st = torch.cuda.current_stream().cuda_stream
        d_len = torch.from_numpy(self.lens).cuda()
        ws = int(lib.ctcb_brnn_sweep_workspace_bytes(H, B))
        # error words and counters 0, the tensor-core operand stacks and rings NaN bytes (written before they are
        # read), 256 NaN bytes behind
        scratch = torch.full((ws + 256,), 255, dtype=torch.uint8, device="cuda")
        scratch[:4096] = 0
        p_all, pre = _buf(torch, self.pre)
        Ww = [_buf(torch, w) for w in self.Ws]
        p = lambda t: None if t is None else t.data_ptr()          # noqa: E731
        W = [x[1] for x in Ww] + [None]
        wholes = [p_all] + [x[0] for x in Ww]
        err = []
        if fwd is None:
            ow = [_buf(torch, np.full((T, B, H), np.nan, np.float32)) for _ in range(nd)]
            o = [x[1] for x in ow] + [None]
            check(lib.ctcb_brnn_sweep_f32(0, T, B, H, p(d_len), p(pre), p(W[0]), p(W[1]), p(o[0]), p(o[1]),
                                          None, None, MAXACT, p(scratch), ws, st))
            torch.cuda.synchronize()
            err.append(scratch[:64].view(torch.int32).cpu().numpy().copy())
            F = [x.cpu().numpy() for x in o[:nd]]
            wholes += [x[0] for x in ow]
            acts = [f.copy() for f in F]
            if self.act == "edges":
                acts = [_edge_states(a, self.lens, seed=7 + i) for i, a in enumerate(acts)]
        else:
            F, acts = fwd["F"], fwd["act"]
        aw = [_buf(torch, a) for a in acts]
        a_ = [x[1] for x in aw] + [None]
        dw = _buf(torch, self.d if d is None else d)
        gw = [_buf(torch, np.full((T, B, H), np.nan, np.float32)) for _ in range(nd)]
        g = [x[1] for x in gw] + [None]
        check(lib.ctcb_brnn_sweep_f32(1, T, B, H, p(d_len), p(dw[1]), p(W[0]), p(W[1]), p(g[0]), p(g[1]),
                                      p(a_[0]), p(a_[1]), MAXACT, p(scratch), ws, st))
        torch.cuda.synchronize()
        err.append(scratch[:64].view(torch.int32).cpu().numpy().copy())
        wholes += [x[0] for x in aw] + [dw[0]] + [x[0] for x in gw]
        tail = scratch[ws:].cpu().numpy()
        guards = all(_guards_intact(w) for w in wholes) and bool((tail == 255).all())
        return dict(F=F, act=acts, dF=[x.cpu().numpy() for x in g[:nd]], err=[int(np.abs(e).max()) for e in err],
                    guards=guards)


def _same_run(r, s):
    return all(_same(x, y) for k in ("F", "dF") for x, y in zip(r[k], s[k]))


# boundary values of the clip and of the BPTT mask 0 < act < maxAct
EDGES = np.array([0.0, -0.0, MAXACT, np.nextafter(np.float32(MAXACT), np.float32(0)),
                  np.nextafter(np.float32(MAXACT), np.float32(100)), np.float32(2.0 ** -126), -np.float32(2.0 ** -126)],
                 np.float32)


def _edge_states(a, lens, seed):
    """States a with a random eighth of the live entries replaced by the mask's boundary values."""
    rng = np.random.RandomState(seed)
    a = a.copy()
    T, B, H = a.shape
    live = np.arange(T)[:, None, None] < np.asarray(lens)[None, :, None]
    pick = live & (rng.rand(T, B, H) < 0.125)
    a[pick] = EDGES[rng.randint(0, len(EDGES), size=int(pick.sum()))]
    return a


# ------------------------------------------------------------------------------------------------ float64
def _tf32(x):
    """x rounded to float32, then its low 13 mantissa bits cleared: the hi part the kernels feed the tensor cores."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xffffe000)
    return u.view(np.float32).astype(np.float64)


def _steps(sw, outs, inputs, Ms, acts, C):
    """Largest |y - y64| / (u S) over the live frames of every direction (y64 the float64 step from the GPU's own y of
    the step before), and of the TF32 emulation's step; asserts the exact properties of each step on the way."""
    T, lens, nd = sw.T, sw.lens, sw.ndir
    bptt = acts is not None
    worst = dict(ratio=0.0, tf32=0.0, exact_steps=0)
    x_in = inputs.astype(np.float64)
    for d in range(nd):
        M = Ms[d].astype(np.float64)            # y_t = f(x_t + y_prev @ M)
        aM, Mtf = np.abs(M), _tf32(Ms[d])
        y = outs[d]
        ascending = (d == 0) != bptt
        order = range(T) if ascending else range(T - 1, -1, -1)
        prev = np.zeros(y.shape[1:])
        for t in order:
            live = t < lens
            yt = y[t].astype(np.float64)
            if live.any():
                xt = x_in[t]
                z = xt + prev.dot(M)
                S = np.abs(xt) + np.abs(prev).dot(aM)
                ztf = xt + _tf32(prev).dot(Mtf)
                if bptt:
                    act = acts[d][t].astype(np.float64)
                    keep = (act > 0) & (act < MAXACT)
                    y64, ytf = np.where(keep, z, 0.0), np.where(keep, ztf, 0.0)
                    masked = ~keep & live[:, None]
                    assert not np.any(y[t].view(np.uint32)[masked]), "a masked element is not +0.0 (t=%d)" % t
                else:
                    y64, ytf = np.clip(z, 0.0, MAXACT), np.clip(ztf, 0.0, MAXACT)
                    lo = (z < -C * U32 * S) & live[:, None]
                    hi = (z > MAXACT + C * U32 * S) & live[:, None]
                    assert np.all(yt[lo] == 0.0), "not exactly clipped at 0 (t=%d)" % t
                    assert np.all(yt[hi] == MAXACT), "not exactly clipped at maxAct (t=%d)" % t
                zero = live & ~np.any(prev, axis=1)       # no recurrent term: the step is exact
                if zero.any():
                    want = y64[zero]
                    assert np.array_equal(yt[zero], want), "y != f(x) exactly after an all-zero state (t=%d)" % t
                    worst["exact_steps"] += int(zero.sum())
                e = np.abs(yt - y64)[live]
                Sl = S[live]
                assert np.all(e[Sl == 0] == 0), "inexact where S = 0 (t=%d)" % t
                pos = Sl > 0
                if pos.any():
                    worst["ratio"] = max(worst["ratio"], float(np.max(e[pos] / (U32 * Sl[pos]))))
                    etf = np.abs(ytf - y64)[live]
                    worst["tf32"] = max(worst["tf32"], float(np.max(etf[pos] / (U32 * Sl[pos]))))
            prev = yt
    return worst


def _check_forward(r, sw, C):
    return _steps(sw, r["F"], sw.pre, [w.T for w in sw.Ws], None, C)


def _check_bptt(r, sw, C):
    return _steps(sw, r["dF"], sw.d, sw.Ws, r["act"], C)


def _check_exact(r, sw):
    """Padded frames +0.0 (outputs start as NaN), everything else finite, guard bands intact, error words 0."""
    assert not any(r["err"]), "error words set: %s" % (r["err"],)
    assert r["guards"], "a guard band or the scratch behind the workspace changed: the sweep wrote outside its arrays"
    pad = np.arange(sw.T)[:, None] >= sw.lens[None, :]
    for x in r["F"] + r["dF"]:
        assert not np.any(x.view(np.uint32)[pad]), "a padded frame is not +0.0"
        assert np.isfinite(x).all(), "an output was not written"


# ------------------------------------------------------------------------------------------------ inputs
def _problem(torch, H, B, T, ndir, seed, lens="ragged", vals="clip", dmode="randn"):
    rng = np.random.RandomState(seed)
    f32 = lambda x: np.asarray(x, dtype=np.float32)                           # noqa: E731
    s = 0.9 / np.sqrt(H / 3.0)                                               # spectral radius ~0.9: well conditioned
    Ws = [f32(rng.uniform(-s, s, (H, H))) for _ in range(ndir)]
    pre = rng.randn(T, B, H) * 2.0 + 0.5
    for t in ([T // 2] if T < 60 else range(T // 6, T, T // 6)):           # drive a third of the units into the clip
        pre[t] += 25.0 * (rng.rand(B, H) < 0.3)
    if lens == "ragged":
        L = rng.randint(max(1, T // 2), T + 1, size=B)
        L[0] = T
        if B > 1:
            L[-1] = 1
    elif lens == "short":                        # every utterance shorter than T: all-padding first backward steps
        L = rng.randint(1, max(2, T - 1), size=B)
    elif lens == "zero":                         # some utterances have no frame at all
        L = rng.randint(1, T + 1, size=B)
        L[0] = T
        L[1::3] = 0
    else:
        L = np.full(B, T)
    pre = f32(pre)
    if vals == "edges":
        # a frame that drives every state below 0; after it, and at each direction's first frame, the state before is
        # all zero and the outputs are exactly clip(pre): put a quarter of them on the clip's kinks
        if T >= 3:
            pre[T // 2] = -1e4
        frames = [(0, slice(None))] + ([(T // 2 + 1, slice(None))] if T >= 3 else [])
        frames += [(int(L[u]) - 1, u) for u in range(B) if L[u] > 0]
        for t, u in frames:
            row = pre[t, u]
            pick = rng.rand(*row.shape) < 0.25
            row[pick] = EDGES[rng.randint(0, len(EDGES), size=int(pick.sum()))]
            pre[t, u] = row
    d = rng.randn(T, B, H)
    if dmode == "last":                          # d only at the last frame of each direction's order
        keep = np.zeros((T, B), bool)
        for u in range(B):
            if L[u] > 0:
                keep[L[u] - 1, u] = True
                if ndir == 2:
                    keep[0, u] = True
        d = d * keep[:, :, None]
    return Sweep(torch, L, pre, Ws, f32(d), act="edges" if vals == "edges" else "own")


# ------------------------------------------------------------------------------------------------ one case
def _sweep_case(name, H, B, T, ndir, expect, torch, lens="ragged", vals="clip", dmode="randn"):
    plan = _check_plan(H, B, ndir, expect, torch)
    _note(plan, B)
    SEEN["cases"] += 1
    C = _bound(plan, H)
    t0 = time.time()
    sw = _problem(torch, H, B, T, ndir, 1000 * H + B + T, lens, vals, dmode)
    r = sw.run()
    _check_exact(r, sw)
    again = sw.run()
    assert _same_run(r, again), "a rerun gave other bytes"
    nz = np.concatenate([np.abs(x[x != 0]) for x in r["dF"]] + [np.abs(sw.d[sw.d != 0])])
    dmin = float(nz.min()) if nz.size else 0.0
    linear = dmin >= TINY
    if linear:
        scaled = sw.run(d=sw.d * SCALE, fwd=r)
        _check_exact(scaled, sw)
        assert all(_same(x, y * SCALE) for x, y in zip(scaled["dF"], r["dF"])), "dF is not exactly linear in d"
    fwd = _check_forward(r, sw, C)
    bptt = _check_bptt(r, sw, C)
    print(json.dumps({"sweep": name, "H": H, "B": B, "T": T, "ndir": ndir, "lens": lens, "vals": vals, "d": dmode,
                      "plan": plan, "C": C, "fwd": fwd["ratio"], "bptt": bptt["ratio"], "tf32_fwd": fwd["tf32"],
                      "tf32_bptt": bptt["tf32"], "exact_steps": fwd["exact_steps"] + bptt["exact_steps"],
                      "rerun_same": True, "linearity_checked": linear, "seconds": round(time.time() - t0, 2)}))
    if vals in ("clip", "edges"):
        assert any((x == MAXACT).any() for x in r["F"]), "the clip is never reached"
    assert fwd["ratio"] <= C and bptt["ratio"] <= C, (fwd, bptt, C)
    if T >= 2:
        assert fwd["tf32"] >= TF32_MARGIN * C and bptt["tf32"] >= TF32_MARGIN * C, (fwd, bptt, C)
    return r, sw, plan


# ------------------------------------------------------------------------------------------------ the shapes of the
# original suite: each on the plan the device chooses by default
@pytest.mark.parametrize("H,B,T", [(128, 8, 40), (128, 3, 33), (256, 9, 25), (512, 4, 30), (512, 32, 50),
                                     (1024, 16, 12), (96, 5, 20), (30, 2, 10), (64, 17, 21), (512, 16, 20),
                                     (256, 64, 10),
                                     # the tensor-core kernel (sweep_tc.cu, H >= 1024): one and two utterance splits, partial
                                     # 16-utterance tiles, the C3 / C4 per-GPU batch widths, H not a power of two
                                     (1024, 128, 10), (1024, 40, 9), (1024, 3, 7), (2048, 32, 8), (2048, 256, 5),
                                     (1536, 20, 6), (1024, 200, 5), (2048, 100, 4)])
def test_sweep_forward_and_bptt(H, B, T, cuda):
    if H >= 1024 and _natural_family(H) == TC:     # these sizes must run on the tensor-core kernel
        from _ctcb import lib
        assert lib.ctcb_sweep_uses_tensor_cores(H, B) == 1, (H, B)
    _sweep_case("%d-%d-%d" % (H, B, T), H, B, T, 2, {"kernel": _natural_family(H)}, cuda)


def test_general_barrier_kernel_when_forced(gknobs, cuda):
    """CTCB_SWEEP=barrier forces the L2/counter-barrier kernel for sizes the cluster kernel would take."""
    gknobs("CTCB_SWEEP", "barrier")
    for H, B, T in ((512, 32, 50), (128, 3, 33), (256, 9, 25)):
        assert _natural_family(H) == GEN, H
        test_sweep_forward_and_bptt(H, B, T, cuda)


# ------------------------------------------------------------------------------------------------ the plan matrix
def _c(name, H, B, T, ndir, forced=None, lens="ragged", vals="clip", dmode="randn", **expect):
    return pytest.param(H, B, T, ndir, forced or {}, dict(lens=lens, vals=vals, dmode=dmode), expect, id=name)


BAR, RR, TC0 = {"CTCB_SWEEP": "barrier"}, {"CTCB_SWEEP": "reread"}, {"CTCB_SWEEP_TC": "0"}
PLAN_CASES = [
    # tensor-core, both directions: every wgmma N at H = 1024 (NP >= 160: the partial aliases the ring)
    _c("tc-np32", 1024, 20, 6, 2, kernel=TC, CS=4, NS=1, NP=32, partial_own=1),
    _c("tc-np64", 1024, 50, 6, 2, kernel=TC, CS=4, NP=64, partial_own=1),
    _c("tc-np96", 1024, 90, 6, 2, kernel=TC, CS=4, NP=96, partial_own=1),
    _c("tc-np128", 1024, 128, 5, 2, kernel=TC, CS=4, NP=128, partial_own=1),
    _c("tc-np160", 1024, 150, 5, 2, kernel=TC, CS=4, NP=160, partial_own=0),
    _c("tc-np192", 1024, 180, 5, 2, kernel=TC, CS=4, NP=192, partial_own=0),
    _c("tc-np224", 1024, 210, 4, 2, kernel=TC, CS=4, NP=224, partial_own=0),
    _c("tc-np256", 1024, 256, 4, 2, kernel=TC, CS=4, NP=256, partial_own=0),
    # cluster sizes: CS = 2 where four-CTA clusters cannot hold the batch, and both smaller sizes forced
    _c("tc-cs2-b300", 1024, 300, 4, 2, kernel=TC, CS=2),
    _c("tc-cs2-forced", 1024, 100, 5, 2, {"CTCB_SWEEP_TC_CS": "2"}, kernel=TC, CS=2),
    _c("tc-cs1-forced", 1024, 40, 5, 2, {"CTCB_SWEEP_TC_CS": "1"}, kernel=TC, CS=1),
    _c("tc-cs1-h1280-uni", 1280, 800, 3, 1, kernel=TC, CS=1, NS=13, NP=64),
    # several utterance splits, the last one holding a single utterance
    _c("tc-h2048-b33", 2048, 33, 5, 2, kernel=TC, NS=2, NP=32),
    # M tiles not a power of two
    _c("tc-h1280", 1280, 40, 5, 2, kernel=TC),
    # tensor-core, forward direction alone (Wb = NULL)
    _c("tc-uni-h1024-np32", 1024, 32, 6, 1, kernel=TC, CS=4, NP=32),
    _c("tc-uni-h1024-np256", 1024, 700, 3, 1, kernel=TC, CS=4, NP=256),
    _c("tc-uni-h2048-np32", 2048, 32, 5, 1, kernel=TC, CS=4, NP=32),
    _c("tc-uni-h2048-np256", 2048, 256, 4, 1, kernel=TC, CS=4, NP=256),
    # edges: one to three frames (T = 1 issues no MMA job at all), a long sweep through the clip several times
    _c("tc-t1", 1024, 16, 1, 2, kernel=TC),
    _c("tc-t2", 1024, 16, 2, 2, kernel=TC),
    _c("tc-t3", 1024, 16, 3, 2, kernel=TC),
    _c("tc-uni-t2", 2048, 8, 2, 1, kernel=TC),
    _c("tc-long-t300", 1024, 16, 300, 2, kernel=TC),
    _c("tc-h512-opt-in", 512, 24, 6, 2, {"CTCB_SWEEP_TC": "2"}, kernel=TC),
    _c("tc-plain-cluster-launch", 1024, 64, 6, 2, {"CTCB_SWEEP_TC_COOP": "0"}, kernel=TC, CS=4, NP=64),
    # ... with one utterance, lengths 0, every utterance shorter than T, the clip's kinks, d at the last frame only
    _c("tc-b1", 1024, 1, 5, 2, kernel=TC, NP=32),
    _c("tc-lens-zero", 1024, 40, 6, 2, lens="zero", kernel=TC),
    _c("tc-short", 2048, 20, 7, 2, lens="short", kernel=TC),
    _c("tc-edges", 1024, 24, 7, 2, vals="edges", kernel=TC),
    _c("tc-d-last", 1024, 24, 9, 2, dmode="last", kernel=TC),
    _c("tc-plain-cs1-np256", 1280, 800, 3, 1, {"CTCB_SWEEP_TC_COOP": "0"}, kernel=TC, CS=1),
    _c("tc-plain-cs2", 1024, 300, 3, 2, {"CTCB_SWEEP_TC_COOP": "0"}, kernel=TC, CS=2),
    # cluster kernel at H = 512 (an H100 holds 14 clusters of 8 CTAs): every group size, B not a multiple of it, one and
    # two directions
    _c("cl-nb1", 512, 7, 8, 2, kernel=CL, NB=1),
    _c("cl-nb2", 512, 27, 8, 1, kernel=CL, NB=2),
    _c("cl-nb3", 512, 20, 8, 2, kernel=CL, NB=3),
    _c("cl-nb4", 512, 55, 8, 1, kernel=CL, NB=4),
    _c("cl-nb5", 512, 33, 8, 2, kernel=CL, NB=5),
    _c("cl-nb6", 512, 83, 6, 1, kernel=CL, NB=6),
    _c("cl-nb7", 512, 47, 8, 2, kernel=CL, NB=7),
    _c("cl-nb8", 512, 55, 8, 2, kernel=CL, NB=8),
    _c("cl-nb7-forced", 512, 9, 8, 2, {"CTCB_SWEEP_NB": "7"}, kernel=CL, NB=7),
    # ... and the switch to the generic kernel once one wave of clusters cannot hold the batch
    _c("cl-to-generic", 512, 57, 6, 2, kernel=GEN, KI=16),
    # cluster kernel at H = 128 and 256, and its edges: T = 1, 2, 3 (the barriers armed for step s + 2 < T, both
    # parities), T = 1000 at the C2 shape and at H = 128, one utterance, lengths 0, the clip's kinks, d at the end only
    _c("cl-h128-nb1", 128, 5, 9, 2, kernel=CL, KI=4, NB=1),
    _c("cl-h256-nb3-forced", 256, 22, 7, 2, {"CTCB_SWEEP_NB": "3"}, kernel=CL, KI=8, NB=3),
    _c("cl-t1", 512, 9, 1, 2, kernel=CL),
    _c("cl-t2", 512, 9, 2, 2, kernel=CL),
    _c("cl-t3", 512, 9, 3, 2, kernel=CL),
    _c("cl-t2-h128-uni", 128, 5, 2, 1, kernel=CL),
    _c("cl-t3-h256", 256, 17, 3, 2, kernel=CL),
    _c("cl-c2-t1000", 512, 32, 1000, 2, kernel=CL, NB=5),
    _c("cl-h128-t1000", 128, 6, 1000, 2, kernel=CL, KI=4),
    _c("cl-b1", 512, 1, 6, 2, kernel=CL, NB=1),
    _c("cl-lens-zero", 256, 20, 8, 2, lens="zero", kernel=CL),
    _c("cl-short", 512, 12, 9, 2, lens="short", kernel=CL),
    _c("cl-edges", 512, 16, 9, 2, vals="edges", kernel=CL),
    _c("cl-edges-h128", 128, 9, 9, 1, vals="edges", kernel=CL),
    _c("cl-d-last", 512, 12, 20, 2, dmode="last", kernel=CL),
    # generic kernel: every register-resident width and the re-reading one, one and two directions
    _c("gen-ki4-uni", 128, 9, 8, 1, BAR, kernel=GEN, KI=4),
    _c("gen-ki8", 256, 20, 8, 2, BAR, kernel=GEN, KI=8),
    _c("gen-ki16-uni", 512, 12, 8, 1, BAR, kernel=GEN, KI=16),
    _c("gen-ki0-h96-uni", 96, 11, 9, 1, kernel=GEN, KI=0),
    _c("gen-ki0-h30", 30, 6, 9, 2, kernel=GEN, KI=0),
    # ... and at H >= 1024 once the batch is wider than any tensor-core plan
    _c("gen-ki32-h1024", 1024, 600, 3, 2, kernel=GEN, KI=32),
    _c("gen-ki32-h1024-uni", 1024, 1100, 3, 1, kernel=GEN, KI=32),
    _c("gen-ki0-h2048", 2048, 300, 3, 2, kernel=GEN, KI=0),
    # ... the re-read path at register widths, odd widths, T = 1, 2, 3, T = 1000, B = 1 and B = 1 (mod 8), a partition
    # without a tile and one partition walking 16 tiles whose last is partial, lengths 0, the kinks, d at the end only
    _c("gen-reread-h128", 128, 9, 6, 2, RR, kernel=GEN, KI=0),
    _c("gen-reread-h1024-uni", 1024, 9, 5, 1, dict(RR, **TC0), kernel=GEN, KI=0),
    _c("gen-h33", 33, 9, 7, 2, kernel=GEN, KI=0),
    _c("gen-h1000", 1000, 17, 5, 2, kernel=GEN, KI=0),
    _c("gen-h1280-uni", 1280, 9, 4, 1, TC0, kernel=GEN, KI=0),
    _c("gen-t1", 256, 9, 1, 2, BAR, kernel=GEN, KI=8),
    _c("gen-t2", 128, 9, 2, 2, BAR, kernel=GEN, KI=4),
    _c("gen-t3", 33, 9, 3, 1, kernel=GEN, KI=0),
    _c("gen-t3-h1024", 1024, 9, 3, 2, TC0, kernel=GEN, KI=32),
    _c("gen-t1000", 128, 6, 1000, 2, BAR, kernel=GEN, KI=4),
    _c("gen-b1", 96, 1, 6, 2, kernel=GEN, KI=0),
    _c("gen-b1-h512", 512, 1, 6, 2, BAR, kernel=GEN, KI=16),
    _c("gen-b-1mod8", 512, 33, 6, 2, BAR, kernel=GEN, KI=16),
    _c("gen-parts4-empty", 256, 37, 6, 2, dict(BAR, CTCB_SWEEP_PARTS="4"), kernel=GEN, KI=8, parts=4),
    _c("gen-parts1-16tiles", 512, 121, 5, 2, dict(BAR, CTCB_SWEEP_PARTS="1"), kernel=GEN, KI=16, parts=1),
    _c("gen-parts1-16tiles-reread", 70, 121, 4, 1, {"CTCB_SWEEP_PARTS": "1"}, kernel=GEN, KI=0, parts=1),
    _c("gen-lens-zero", 96, 20, 8, 2, lens="zero", kernel=GEN),
    _c("gen-short", 256, 12, 9, 2, BAR, lens="short", kernel=GEN),
    _c("gen-edges", 96, 16, 9, 2, vals="edges", kernel=GEN),
    _c("gen-edges-ki16", 512, 16, 9, 2, BAR, vals="edges", kernel=GEN),
    _c("gen-d-last", 1000, 12, 20, 2, dmode="last", kernel=GEN),
]


@pytest.mark.parametrize("H,B,T,ndir,forced,recipe,expect", PLAN_CASES)
def test_sweep_plan(H, B, T, ndir, forced, recipe, expect, request, gknobs, cuda):
    name = request.node.callspec.id
    for k, v in forced.items():
        gknobs(k, v)
    if expect["kernel"] == GEN and H >= 1024 and "CTCB_SWEEP_TC" not in forced:
        from _ctcb import lib
        assert ndir == 1 or lib.ctcb_sweep_uses_tensor_cores(H, B) == 0
    _sweep_case(name, H, B, T, ndir, expect, cuda, **recipe)


# ------------------------------------------------------------------------------------------------ plan independence
@pytest.mark.parametrize("H", [128, 256, 512])
def test_cluster_bits_do_not_depend_on_nb(H, gknobs, cuda):
    """The cluster kernel's per-utterance arithmetic does not depend on NB: every forced NB = 1..8 gives the bytes of
    the automatic plan.  B = 841 = 1 (mod NB) for every NB, so the last cluster's invalid owners send zeros."""
    torch = cuda
    B, T = 841, 5
    sw = _problem(torch, H, B, T, 2, seed=5 * H)
    gknobs("CTCB_SWEEP_NB", "1")
    plan1 = _check_plan(H, B, 2, {"kernel": CL, "NB": 1}, torch)
    ref = sw.run()
    _check_exact(ref, sw)
    C = _bound(plan1, H)
    fwd, bptt = _check_forward(ref, sw, C), _check_bptt(ref, sw, C)
    assert fwd["ratio"] <= C and bptt["ratio"] <= C, (fwd, bptt)
    _note(plan1, B)
    for nb in range(2, 9):
        gknobs("CTCB_SWEEP_NB", str(nb))
        plan = _check_plan(H, B, 2, {"kernel": CL, "KI": H // 32, "NB": nb}, torch)
        r = sw.run()
        _check_exact(r, sw)
        _note(plan, B)
        assert _same_run(r, ref), "NB=%d gave other bytes than NB=1" % nb
    print(json.dumps({"sweep_bits_cluster_h%d" % H: dict(B=B, T=T, nb="1..8", fwd=fwd["ratio"], bptt=bptt["ratio"])}))


@pytest.mark.parametrize("H", [128, 256, 512, 1024])
def test_generic_bits_do_not_depend_on_partitions_or_ki(H, gknobs, cuda):
    """The generic kernel's register and re-read paths accumulate in the same lane order (k = lane + 32 i) and
    partitions change no arithmetic: every forced partition count and the re-read path give the bytes of the
    automatic plan.  B = 121: 16 tiles, the last of one utterance; 1 partition walks all 16, 5 and 7 leave one empty."""
    torch = cuda
    B, T = 121, 5
    sms = _sms(torch)
    gknobs("CTCB_SWEEP", "barrier")
    gknobs("CTCB_SWEEP_TC", "0")
    sw = _problem(torch, H, B, T, 2, seed=7 * H)
    auto = _check_plan(H, B, 2, {"kernel": GEN, "KI": H // 32}, torch)
    ref = sw.run()
    _check_exact(ref, sw)
    C = _bound(auto, H)
    fwd, bptt = _check_forward(ref, sw, C), _check_bptt(ref, sw, C)
    assert fwd["ratio"] <= C and bptt["ratio"] <= C, (fwd, bptt)
    _note(auto, B)
    runs = {"auto": auto}
    for reread in (False, True):
        gknobs("CTCB_SWEEP", "reread" if reread else "barrier")
        gknobs("CTCB_SWEEP_PARTS", "auto")
        cap = _plan(H, 8 * 500, 2)["parts"]
        for parts in [None] + sorted({1, 2, 3, 5, 7, cap}):
            if parts is not None and parts > cap or (parts is None and not reread):
                continue
            gknobs("CTCB_SWEEP_PARTS", str(parts) if parts else "auto")
            want = _expect_generic(H, B, 2, sms, reread, parts)
            plan = _check_plan(H, B, 2, {"kernel": GEN, "KI": 0 if reread else H // 32}, torch)
            assert plan == dict(want, CS=0), (plan, want)
            r = sw.run()
            _check_exact(r, sw)
            _note(plan, B)
            label = "%s-parts%s" % ("reread" if reread else "ki", parts or "auto")
            runs[label] = plan
            assert _same_run(r, ref), "%s gave other bytes than the automatic plan %s" % (label, auto)
    print(json.dumps({"sweep_bits_generic_h%d" % H: runs}))


def _sub(sw, n):
    """The first n utterances of problem sw."""
    return Sweep(sw.torch, sw.lens[:n], np.ascontiguousarray(sw.pre[:, :n]), sw.Ws,
                 np.ascontiguousarray(sw.d[:, :n]))


@pytest.mark.parametrize("H,ndir", [(1024, 1), (1024, 2), (2048, 2)])
def test_tensor_core_bits_do_not_depend_on_the_split(H, ndir, gknobs, cuda):
    """Each utterance column of the tensor-core kernel is its own: the first utterances of a batch get the same bytes
    whatever the batch, and so the number of utterance splits (NS) and the wgmma N (NP) of the plan.  The K-slice
    count CS changes the split-K reduction and is held fixed."""
    torch = cuda
    B, T = 256, 5
    sw = _problem(torch, H, B, T, ndir, seed=11 * H + ndir)
    cs = _plan(H, B, ndir)["CS"]
    gknobs("CTCB_SWEEP_TC_CS", str(cs))
    full = sw.run()
    _check_exact(full, sw)
    plans = {}
    for n in (1, 16, 17, 32, 33, 64, 100, 128, 200, 256):
        plan = _plan(H, n, ndir)
        if plan["kernel"] != TC or plan["CS"] != cs:
            continue
        _note(plan, n)
        sub = _sub(sw, n)
        r = sub.run() if n < B else full
        _check_exact(r, sub)
        same = all(_same(np.ascontiguousarray(x[:, :n]), y) for k in ("F", "dF") for x, y in zip(full[k], r[k]))
        plans["B%d" % n] = dict(NS=plan["NS"], NP=plan["NP"], same=same)
        assert same, "B=%d (NS=%d, NP=%d) gave other bytes for its utterances than B=%d" % (n, plan["NS"], plan["NP"], B)
    print(json.dumps({"sweep_bits_tc_h%d_%s" % (H, "bi" if ndir == 2 else "uni"): dict(CS=cs, runs=plans)}))


def _uni_of_direction(sw, d):
    """The uni-directional problem that direction d of bi-directional problem sw is: W_d and, for d = 1, every
    utterance's pre-activations and deltas reversed within its own length."""
    pre, dd = sw.pre.copy(), sw.d.copy()
    if d == 1:
        pre, dd = _reverse(pre, sw.lens), _reverse(dd, sw.lens)
    return Sweep(sw.torch, sw.lens, pre, [sw.Ws[d]], dd)


def _reverse(x, lens):
    y = x.copy()
    for u, Tu in enumerate(lens):
        y[:Tu, u] = x[:Tu, u][::-1]
    return y


@pytest.mark.parametrize("H,B,forced", [(30, 13, {}), (96, 9, {}), (128, 13, {}), (512, 9, {}), (256, 17, BAR),
                                          (1024, 9, TC0), (1024, 24, {}), (2048, 20, {"CTCB_SWEEP_TC_CS": "2"})],
                         ids=["gen-h30", "gen-h96", "cl-h128", "cl-h512", "gen-h256", "gen-h1024", "tc-h1024",
                              "tc-h2048-cs2"])
def test_each_direction_is_a_uni_directional_sweep(H, B, forced, gknobs, cuda):
    """Each direction of a bi-directional launch gives the bytes of a uni-directional launch on that direction's W,
    direction 1 with every utterance reversed within its own length (padded frames stay where they are); the
    tensor-core plans of both launches take the same K-slice count."""
    torch = cuda
    for k, v in forced.items():
        gknobs(k, v)
    T = 7
    sw = _problem(torch, H, B, T, 2, seed=13 * H + B)
    bi = _plan(H, B, 2)
    r = sw.run()
    _check_exact(r, sw)
    for d in range(2):
        usw = _uni_of_direction(sw, d)
        uni = _plan(H, B, 1)
        assert uni["kernel"] == bi["kernel"] and (bi["kernel"] != TC or uni["CS"] == bi["CS"]), (bi, uni)
        u = usw.run()
        _check_exact(u, usw)
        for k in ("F", "dF"):
            got = r[k][d] if d == 0 else _reverse(r[k][d], sw.lens)
            assert _same(got, u[k][0]), "direction %d %s differs from a uni launch (%s / %s)" % (d, k, bi, uni)


# ------------------------------------------------------------------------------------------------ refusals
def _sweep_call(torch, H, B, ndir, T=1):
    """One forward sweep call at (H, B, ndir) on small inputs: (rc, message, launches)."""
    from _ctcb import lib
    st = torch.cuda.current_stream().cuda_stream
    ws = int(lib.ctcb_brnn_sweep_workspace_bytes(H, B))
    scratch = torch.zeros(ws, dtype=torch.uint8, device="cuda")
    pre = torch.zeros(T, B, H, device="cuda")
    W = [torch.zeros(H, H, device="cuda") for _ in range(ndir)] + [None]
    out = [torch.zeros(T, B, H, device="cuda") for _ in range(ndir)] + [None]
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    p = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    n0 = lib.ctcb_launch_count()
    rc = lib.ctcb_brnn_sweep_f32(0, T, B, H, p(lens), p(pre), p(W[0]), p(W[1]), p(out[0]), p(out[1]), None, None,
                                 MAXACT, p(scratch), ws, st)
    msg = lib.ctcb_last_error().decode()
    torch.cuda.synchronize()
    return rc, msg, lib.ctcb_launch_count() - n0


def _create_rc(H, maxB, ndir):
    import _ctcb
    from _ctcb import lib
    cfg = _ctcb.BrnnConfig(41, 32, H, 3, 2, 50, maxB, 10, 0.0, 20.0, int(ndir == 1), 1, 0)
    h = ctypes.c_void_p()
    rc = lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h))
    msg = lib.ctcb_last_error().decode()
    if rc == 0:
        lib.ctcb_brnn_destroy(h)
    return rc, msg


def _next_call_succeeds(torch):
    """A tensor-core sweep (kernel launches checked with cudaGetLastError) and a generic one succeed: no runtime error
    was left pending by a refusal."""
    for H in (1024, 96):
        rc, msg, n = _sweep_call(torch, H, 4, 2, T=2)
        assert rc == 0 and n >= 1, (H, rc, msg)


def _widest(ndir):
    """The widest H the generic plan holds under the knobs in effect (feasibility falls with H)."""
    lo, hi = 32, 8192
    assert _plan_rc(lo, 3, ndir)[0] == 0 and _plan_rc(hi, 3, ndir)[0] != 0
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _plan_rc(mid, 3, ndir)[0] == 0 else (lo, mid)
    return lo


@pytest.mark.parametrize("ndir", [1, 2])
def test_the_widest_generic_layer_runs_and_the_next_is_refused(ndir, gknobs, cuda):
    """The widest H whose generic sweep the device holds co-resident runs and matches float64; one unit more is refused
    with CTCB_EINVAL by the sweep (without a launch), by ctcb_debug_sweep_plan and by ctcb_brnn_create, and the next
    library call succeeds.  The tensor-core plan is off, so the generic kernel is what runs."""
    torch = cuda
    gknobs("CTCB_SWEEP_TC", "0")
    Hmax = _widest(ndir)
    want = _expect_generic(Hmax, 3, ndir, _sms(torch))
    assert want is not None and _expect_generic(Hmax + 1, 3, ndir, _sms(torch)) is None, Hmax
    if _sms(torch) == H100_SMS:
        assert Hmax == {1: 4224, 2: 3612}[ndir], Hmax
    r, sw, plan = _sweep_case("widest-%s" % ("bi" if ndir == 2 else "uni"), Hmax, 3, 3, ndir, {"kernel": GEN}, torch,
                              lens="full")
    rc, plan1 = _plan_rc(Hmax + 1, 3, ndir)
    assert rc == -1, rc
    rc, msg, n = _sweep_call(torch, Hmax + 1, 3, ndir)
    assert rc == -1 and n == 0 and "layerSize %d" % (Hmax + 1) in msg and "co-resident" in msg, (rc, msg, n)
    rc, cmsg = _create_rc(Hmax + 1, 3, ndir)
    assert rc == -1 and "layerSize %d" % (Hmax + 1) in cmsg, (rc, cmsg)
    assert _create_rc(Hmax, 3, ndir)[0] == 0
    _next_call_succeeds(torch)
    print(json.dumps({"sweep_widest_%s" % ("bi" if ndir == 2 else "uni"): dict(plan, H=Hmax, refused=msg)}))


def test_a_layer_beyond_the_shared_memory_opt_in_is_refused(gknobs, cuda):
    """Where the generic kernel's 8 (ceil4(H) + 4) floats of shared memory exceed the per-CTA opt-in maximum, the sweep
    planner and the LSTM planner refuse with CTCB_EINVAL before they ask for the kernel attribute, and leave no
    runtime error pending for the next call."""
    torch = cuda
    from _ctcb import lib
    gknobs("CTCB_SWEEP_TC", "0")
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    H = next(h for h in range(4000, 20000) if _smem(h) > optin)
    assert _smem(H - 1) <= optin
    for ndir in (1, 2):
        rc, _ = _plan_rc(H, 3, ndir)
        assert rc == -1 and "shared memory" in lib.ctcb_last_error().decode(), (rc, lib.ctcb_last_error())
        _next_call_succeeds(torch)
        rc, msg, n = _sweep_call(torch, H, 3, ndir)
        assert rc == -1 and n == 0 and "shared memory" in msg, (rc, msg)
        _next_call_succeeds(torch)
        rc, msg = _create_rc(H, 3, ndir)
        assert rc == -1 and "shared memory" in msg, (rc, msg)
        _next_call_succeeds(torch)
        out = (ctypes.c_int32 * 4)()
        for peep in (0, 1):
            rc = lib.ctcb_debug_lstm_plan(H, 3, ndir, peep, out)
            assert rc == -1 and "shared memory" in lib.ctcb_last_error().decode(), (rc, lib.ctcb_last_error())
            _next_call_succeeds(torch)
    # one unit narrower the attribute is granted and co-residency decides: still CTCB_EINVAL
    rc, msg, n = _sweep_call(torch, H - 1, 3, 1)
    assert rc == -1 and n == 0 and "co-resident" in msg, (rc, msg)
    _next_call_succeeds(torch)
    print(json.dumps({"sweep_smem_refusal": dict(H=H, smem=_smem(H), optin=optin)}))


def test_create_refuses_a_relu_net_the_device_cannot_sweep_at_max_batch(cuda):
    """Bi-directional H = 4096: the tensor-core plan holds B = 128 but not 256 on a 132-SM H100, and the generic kernel
    would need 256 co-resident CTAs of 131 KB; ctcb_brnn_create refuses maxB = 256 with the planner's message."""
    torch = cuda
    if _sms(torch) != H100_SMS:
        pytest.skip("the edge is laid out for 132 SMs")
    assert _plan_rc(4096, 128, 2)[1]["kernel"] == TC
    assert _plan_rc(4096, 256, 2)[0] == -1
    assert _create_rc(4096, 128, 2)[0] == 0
    rc, msg = _create_rc(4096, 256, 2)
    assert rc == -1 and "layerSize 4096" in msg and "co-resident" in msg, (rc, msg)
    _next_call_succeeds(torch)


def test_a_partition_count_the_device_cannot_hold_is_refused(gknobs, cuda):
    """CTCB_SWEEP_PARTS above the generic kernel's capacity is refused before any launch; at the capacity it runs."""
    torch = cuda
    for H, ndir, forced in ((1024, 2, TC0), (512, 2, BAR), (96, 1, {})):
        for k, v in forced.items():
            gknobs(k, v)
        gknobs("CTCB_SWEEP_PARTS", "auto")
        cap = _plan(H, 8 * 500, ndir)["parts"]
        gknobs("CTCB_SWEEP_PARTS", str(cap + 1))
        assert _plan_rc(H, 8 * 500, ndir)[0] == -1
        rc, msg, n = _sweep_call(torch, H, 8 * (cap + 1), ndir)
        assert rc == -1 and n == 0 and "CTCB_SWEEP_PARTS=%d" % (cap + 1) in msg, (rc, msg)
        gknobs("CTCB_SWEEP_PARTS", str(cap))
        assert _plan(H, 8 * (cap + 1), ndir)["parts"] == cap
        rc, msg, n = _sweep_call(torch, H, 8 * (cap + 1), ndir)
        assert rc == 0 and n == 1, (rc, msg)
        gknobs("CTCB_SWEEP_PARTS", "auto")


def test_every_instantiation_and_partition_edge_was_reached(cuda):
    """The cases above reached all five sweep_kernel<KI>, all 24 sweep_cluster_kernel<KI, NB>, every wgmma N of
    sweep_tc_kernel<NP> with and without a partial region of its own, CS = 1, 2 and 4, cooperative and plain cluster
    launches, a generic partition without a tile and one walking 16 tiles whose last is partial."""
    if SEEN["cases"] < len(PLAN_CASES):
        pytest.skip("run with the whole module: %d cases ran" % SEEN["cases"])
    print(json.dumps({"sweep_plans_reached": {k: sorted(v) if isinstance(v, set) else v for k, v in SEEN.items()}}))
    assert SEEN["gen"] == {0, 4, 8, 16, 32}, SEEN["gen"]
    assert SEEN["cl"] == {(ki, nb) for ki in (4, 8, 16) for nb in range(1, 9)}, SEEN["cl"]
    assert SEEN["np"] == set(range(32, 257, 32)) and SEEN["own"] == {0, 1} and SEEN["cs"] == {1, 2, 4}, SEEN
    assert SEEN["coop"] == {"0", "1"}, SEEN["coop"]
    assert SEEN["empty"] > 0 and SEEN["multi16"] > 0, SEEN
