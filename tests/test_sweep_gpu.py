"""GPU unit test of the persistent recurrent sweep on its own (ctcb_brnn_sweep_f32) against a float64 restatement of
brnnet.py:144-152 (forward) and :208-224 (BPTT), vectorised over utterances.

The sweep is a planner over three kernels (the tensor-core kernel for H >= 1024, the cluster kernel for H = 128/256/512,
the generic cooperative kernel for everything else and for batches the others cannot hold).  Every case names the plan it
targets and checks it with ctcb_debug_sweep_plan before launching, so no case passes on a plan it did not mean to test.
Cases that need a planner knob set it in this process (recipes.knobs) and restore it afterwards.

The bound is per kernel family, on  max|gpu - ref| / max(1, max|ref|)  per direction, and it is tight enough to tell the
fp32-faithful 3xTF32 tensor-core arithmetic from plain TF32: each case also runs a TF32 emulation of the same sweep on the
CPU (both operands truncated to 10 mantissa bits as the kernel truncates them, only the hi.hi product kept, accumulated in
float64) and requires it to be at least TF32_MARGIN times the bound away from the float64 result.  Each case prints its
plan, errors, bound and the emulation's error as one JSON line (shown with pytest -s)."""
import json
import time

import numpy as np
import pytest

from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
MAXACT = 20.0
KERNELS = ("generic", "cluster", "tensor-core")
H100_SMS = 132             # the plans below are laid out for the 132-SM H100 SXM; other parts skip a plan they cannot reach
# Bounds on the normalised error above, per kernel family, at most 4x the largest error measured on an H100 80GB HBM3
# (power limit 400 W) over the cases of this file, forward and BPTT.  The FFMA kernels round every product and sum in
# fp32: measured at most 3.6e-7 (generic) and 3.1e-7 (cluster).  The tensor-core kernel's error grows with the chain each
# CTA accumulates on the tensor cores, its K-slice H / CS (the wgmma accumulator does not round to nearest): measured at
# most 2.4e-8 per element of the slice (6.1e-6 at H / CS = 256, 1.8e-5 at 1024), so its bound is TC_BOUND_PER_K * H / CS.
# The TF32 emulation stays at least 11x the bound away in every case.
BOUND = {"generic": 1.2e-6, "cluster": 1.2e-6}
TC_BOUND_PER_K = 4e-8
TF32_MARGIN = 8.0


def _bound(plan, H):
    return TC_BOUND_PER_K * H / plan["CS"] if plan["kernel"] == "tensor-core" else BOUND[plan["kernel"]]


# ------------------------------------------------------------------------------------------------ references
def _tf32(x):
    """x rounded to float32, then its low 13 mantissa bits cleared: the hi part the kernels feed the tensor cores."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xffffe000)
    return u.view(np.float32).astype(np.float64)


def _recur(x, W, order, live, step, tf32):
    """out[t] = step(t, x[t] + out[prev] . W^T) over the times in `order`, zero beyond each utterance's length."""
    out = np.zeros_like(x)
    Wt = (_tf32(W) if tf32 else W).T
    prev = None
    for t in order:
        h = x[t] if prev is None else x[t] + (_tf32(prev) if tf32 else prev) @ Wt
        out[t] = step(t, h) * live[t][:, None]
        prev = out[t]
    return out


def _ref_forward(pre, Wf, Wb, lens, maxAct, tf32=False):
    """For / Back of brnnet.py:144-152 for all utterances at once; Wb None: the forward direction alone."""
    T = pre.shape[0]
    live = np.arange(T)[:, None] < np.asarray(lens)[None, :]
    clip = lambda t, h: np.clip(h, 0.0, maxAct)
    F = _recur(pre, Wf, range(T), live, clip, tf32)
    Bk = None if Wb is None else _recur(pre, Wb, range(T - 1, -1, -1), live, clip, tf32)
    return F, Bk


def _ref_bptt(d, Wf, Wb, F, Bk, lens, maxAct, tf32=False):
    """dFor / dBack of brnnet.py:208-224 for all utterances at once, masked by within(0, maxAct) of the given states."""
    T = d.shape[0]
    live = np.arange(T)[:, None] < np.asarray(lens)[None, :]
    mF = (F > 0) & (F < maxAct)
    dF = _recur(d, Wf.T, range(T - 1, -1, -1), live, lambda t, h: h * mF[t], tf32)
    dB = None
    if Wb is not None:
        mB = (Bk > 0) & (Bk < maxAct)
        dB = _recur(d, Wb.T, range(T), live, lambda t, h: h * mB[t], tf32)
    return dF, dB


def _err(g, r):
    return float(np.abs(g - r).max() / max(1.0, np.abs(r).max()))


# ------------------------------------------------------------------------------------------------ plans
def _plan(H, B, ndir):
    import ctypes
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_sweep_plan(H, B, ndir, out))
    k = out[0]
    plan = dict(kernel=KERNELS[k], KI=out[1], CS=out[2])
    plan[("parts", "NB", "NS")[k]] = out[3]
    if k == 2:
        plan.update(NP=out[4], stages=out[5], partial_own=out[6])
    return plan


def _check_plan(H, B, ndir, expect, torch):
    plan = _plan(H, B, ndir)
    wrong = {k: (v, plan.get(k)) for k, v in expect.items() if plan.get(k) != v}
    if wrong:
        msg = "H=%d B=%d ndir=%d: planned %s, this case targets %s" % (H, B, ndir, plan, expect)
        if torch.cuda.get_device_properties(0).multi_processor_count != H100_SMS:
            pytest.skip("plan not reachable on this device: " + msg)
        pytest.fail(msg)
    return plan


def _natural_family(H):
    """The kernel family the planner picks for a layer size at a small batch, under the knobs in effect."""
    return _plan(H, 1, 2)["kernel"]


# ------------------------------------------------------------------------------------------------ one case
def _sweep_case(name, H, B, T, ndir, expect, torch):
    import _ctcb
    from _ctcb import lib, check, ptr
    plan = _check_plan(H, B, ndir, expect, torch)
    bound = _bound(plan, H)
    t0 = time.time()
    rng = np.random.RandomState(1000 * H + B + T)
    f32 = lambda x: np.asarray(x, dtype=np.float32).astype(np.float64)       # the reference sees the kernel's inputs
    s = 0.9 / np.sqrt(H / 3.0)                                               # spectral radius ~0.9: well conditioned
    Wf = f32(rng.uniform(-s, s, (H, H)))
    Wb = f32(rng.uniform(-s, s, (H, H))) if ndir == 2 else None
    pre = rng.randn(T, B, H) * 2.0 + 0.5
    for t in ([T // 2] if T < 60 else range(T // 6, T, T // 6)):           # drive a third of the units into the clip
        pre[t] += 25.0 * (rng.rand(B, H) < 0.3)
    pre = f32(pre)                                    # padded frames keep their values: the kernel must ignore them
    lens = rng.randint(max(1, T // 2), T + 1, size=B)
    lens[0] = T
    if B > 1:
        lens[-1] = 1
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    d_pre, d_Wf = dev(pre), dev(Wf)
    d_Wb = dev(Wb) if ndir == 2 else None
    d_len = torch.from_numpy(lens.astype(np.int32)).cuda()
    oF = torch.empty(T, B, H, device="cuda")
    oB = torch.empty(T, B, H, device="cuda") if ndir == 2 else None
    nscr = int(lib.ctcb_brnn_sweep_workspace_bytes(H, B))
    scratch = torch.zeros(nscr // 4, dtype=torch.int32, device="cuda")
    st = _ctcb.current_stream()
    check(lib.ctcb_brnn_sweep_f32(0, T, B, H, ptr(d_len), ptr(d_pre), ptr(d_Wf), ptr(d_Wb), ptr(oF), ptr(oB), None,
                                  None, MAXACT, ptr(scratch), nscr, st))
    torch.cuda.synchronize()
    flags_fwd = scratch[:3].tolist()
    gfwd = [o.cpu().numpy().astype(np.float64) for o in (oF, oB) if o is not None]
    rfwd = [r for r in _ref_forward(pre, Wf, Wb, lens, MAXACT) if r is not None]
    efwd = [r for r in _ref_forward(pre, Wf, Wb, lens, MAXACT, tf32=True) if r is not None]

    # BPTT on the float32 states the kernel itself produced (so the masks agree exactly)
    d = f32(rng.randn(T, B, H))
    odF = torch.empty(T, B, H, device="cuda")
    odB = torch.empty(T, B, H, device="cuda") if ndir == 2 else None
    check(lib.ctcb_brnn_sweep_f32(1, T, B, H, ptr(d_len), ptr(dev(d)), ptr(d_Wf), ptr(d_Wb), ptr(odF), ptr(odB),
                                  ptr(oF), ptr(oB), MAXACT, ptr(scratch), nscr, st))
    torch.cuda.synchronize()
    flags_bptt = scratch[:3].tolist()
    gbptt = [o.cpu().numpy().astype(np.float64) for o in (odF, odB) if o is not None]
    states = gfwd + [None] * (2 - ndir)
    rbptt = [r for r in _ref_bptt(d, Wf, Wb, states[0], states[1], lens, MAXACT) if r is not None]
    ebptt = [r for r in _ref_bptt(d, Wf, Wb, states[0], states[1], lens, MAXACT, tf32=True) if r is not None]

    err_fwd = max(_err(g, r) for g, r in zip(gfwd, rfwd))
    err_bptt = max(_err(g, r) for g, r in zip(gbptt, rbptt))
    tf32_fwd = min(_err(e, r) for e, r in zip(efwd, rfwd))
    tf32_bptt = min(_err(e, r) for e, r in zip(ebptt, rbptt))
    print(json.dumps({"sweep": name, "H": H, "B": B, "T": T, "ndir": ndir, "plan": plan,
                      "err_fwd": err_fwd, "err_bptt": err_bptt, "bound": bound,
                      "tf32_err_fwd": tf32_fwd, "tf32_err_bptt": tf32_bptt, "seconds": round(time.time() - t0, 2)}))

    assert flags_fwd == [0, 0, 0] and flags_bptt == [0, 0, 0], "error flags %s %s" % (flags_fwd, flags_bptt)
    pad = np.arange(T)[:, None] >= lens[None, :]
    for g in gfwd + gbptt:
        assert np.isfinite(g).all()
        assert not g[pad].any(), "padded frames are not zero"
    assert (rfwd[0] >= MAXACT).any(), "the clip is never reached"
    for g, r in zip(gfwd, rfwd):
        assert _err(g, r) <= bound, np.argwhere(np.abs(g - r) > bound * max(1.0, np.abs(r).max()))[:5]
    for g, r in zip(gbptt, rbptt):
        assert _err(g, r) <= bound, np.argwhere(np.abs(g - r) > bound * max(1.0, np.abs(r).max()))[:5]
    if T == 1:
        # no recurrence: the sweep is the clip / mask of its input, which every kernel must reproduce exactly (and which
        # the TF32 emulation reproduces exactly too, so there is nothing to separate)
        assert err_fwd == 0.0 and err_bptt == 0.0
    else:
        assert tf32_fwd >= TF32_MARGIN * bound, (tf32_fwd, bound)
        assert tf32_bptt >= TF32_MARGIN * bound, (tf32_bptt, bound)


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
    if H >= 1024 and _natural_family(H) == "tensor-core":     # these sizes must run on the tensor-core kernel
        from _ctcb import lib
        assert lib.ctcb_sweep_uses_tensor_cores(H, B) == 1, (H, B)
    _sweep_case("%d-%d-%d" % (H, B, T), H, B, T, 2, {"kernel": _natural_family(H)}, cuda)


def test_general_barrier_kernel_when_forced(knobs, cuda):
    """CTCB_SWEEP=barrier forces the L2/counter-barrier kernel for sizes the cluster kernel would take."""
    knobs("CTCB_SWEEP", "barrier")
    for H, B, T in ((512, 32, 50), (128, 3, 33), (256, 9, 25)):
        assert _natural_family(H) == GEN, H
        test_sweep_forward_and_bptt(H, B, T, cuda)


# ------------------------------------------------------------------------------------------------ the plan matrix
TC, CL, GEN = "tensor-core", "cluster", "generic"


def _c(name, H, B, T, ndir, forced=None, **expect):
    return pytest.param(H, B, T, ndir, forced or {}, expect, id=name)


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
    # generic kernel: every register-resident width and the re-reading one, one and two directions
    _c("gen-ki4-uni", 128, 9, 8, 1, {"CTCB_SWEEP": "barrier"}, kernel=GEN, KI=4),
    _c("gen-ki8", 256, 20, 8, 2, {"CTCB_SWEEP": "barrier"}, kernel=GEN, KI=8),
    _c("gen-ki16-uni", 512, 12, 8, 1, {"CTCB_SWEEP": "barrier"}, kernel=GEN, KI=16),
    _c("gen-ki0-h96-uni", 96, 11, 9, 1, kernel=GEN, KI=0),
    _c("gen-ki0-h30", 30, 6, 9, 2, kernel=GEN, KI=0),
    # ... and at H >= 1024 once the batch is wider than any tensor-core plan
    _c("gen-ki32-h1024", 1024, 600, 3, 2, kernel=GEN, KI=32),
    _c("gen-ki32-h1024-uni", 1024, 1100, 3, 1, kernel=GEN, KI=32),
    _c("gen-ki0-h2048", 2048, 300, 3, 2, kernel=GEN, KI=0),
]


@pytest.mark.parametrize("H,B,T,ndir,forced,expect", PLAN_CASES)
def test_sweep_plan(H, B, T, ndir, forced, expect, request, knobs, cuda):
    name = request.node.callspec.id
    for k, v in forced.items():
        knobs(k, v)
    if expect["kernel"] == GEN and H >= 1024:
        from _ctcb import lib
        assert ndir == 1 or lib.ctcb_sweep_uses_tensor_cores(H, B) == 0
    _sweep_case(name, H, B, T, ndir, expect, cuda)
