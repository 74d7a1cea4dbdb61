"""GPU unit test of the clipped-ReLU recurrent sweep in TF32 mode (ctcb_brnn_sweep_tf32) on every case of
test_sweep_gpu.py.

The tensor-core kernel in TF32 mode rounds W (W^T for the BPTT) and each step's state to the nearest TF32 value and runs
one MMA per product; S_t itself is the exact fp32 result of the step (include/ctcb200.h).  So each output is checked
step-locally, as test_sweep_gpu.py does, against float64 of the GPU's own previous state and of W, both rounded by rna
(test_gemm_tf32_gpu.py):  |y - y64r| <= (c0 + c1 L) u S,  L = H / CS / 32,  S = |x_t| + |y_{t-1}| |M|.
Negative controls on the same steps must miss y64r by at least MARGIN times that bound: the float64 step of the
truncated operands, and the step the fp32-faithful sweep (ctcb_brnn_sweep_f32) computes from the same inputs, compared
at the first step of each direction that has a recurrent term (where both sweeps start from the same state).
The cluster and generic kernels have no TF32 mode: their plans give ctcb_brnn_sweep_f32's bytes.  Exact properties as
in test_sweep_gpu.py: outputs start as NaN and padded frames come back +0.0, the guard bands and the scratch behind the
workspace are untouched, the error words are 0, a rerun gives the same bytes.  Each case prints its plans and ratios as
one JSON line (pytest -s)."""
import contextlib
import ctypes
import json

import numpy as np
import pytest

import test_sweep_gpu as sg
from recipes import knobs  # noqa: F401  (fixture)
from test_gemm_tf32_gpu import rna, trunc
from test_sweep_gpu import gknobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
# (c0, c1) of the step-local bound of the TF32 kernel: at most 4x the largest ratio measured on an H100 80GB HBM3 (power
# limit 700 W) over the cases of this file, forward and BPTT, at each L: 2.18 at L = 4, 3.80 at L = 8, 3.78 at L = 10,
# 3.81 at L = 12, 8.48 at L = 16 (H = 1024 on clusters of 2, the tightest: bound 1.65x), 13.9 at L = 32, 14.95 at L = 40.
# The controls then measured at least 36 bounds (the fp32-faithful sweep, L = 32) and 108 (truncation).
TF32_C0, TF32_C1 = 6.0, 0.5
MARGIN = 10.0
PLAN_FIELDS = ("kernel", "KI", "CS", "groups", "NP", "stages", "partial_own", "per_sm")


def _raw_plan(fn, H, B, ndir):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(getattr(lib, fn)(H, B, ndir, out))
    return dict(zip(PLAN_FIELDS, list(out)))


@contextlib.contextmanager
def _tf32_entry():
    """Sweep.run of test_sweep_gpu.py with ctcb_brnn_sweep_tf32 in place of ctcb_brnn_sweep_f32."""
    from _ctcb import lib
    f32 = lib.ctcb_brnn_sweep_f32
    lib.ctcb_brnn_sweep_f32 = lib.ctcb_brnn_sweep_tf32
    try:
        yield
    finally:
        lib.ctcb_brnn_sweep_f32 = f32


def _steps_tf32(sw, outs, inputs, Ms, acts, bound, ref_outs):
    """Largest |y - y64r| / (u S) over the live frames; the truncation control's; and the fp32-faithful sweep's
    (ref_outs) at each direction's first step with a recurrent term."""
    T, lens, nd = sw.T, sw.lens, sw.ndir
    bptt = acts is not None
    worst = dict(ratio=0.0, trunc=np.inf, f32=0.0)
    x_in = inputs.astype(np.float64)
    for d in range(nd):
        Mr, Mt = rna(Ms[d]).astype(np.float64), trunc(Ms[d]).astype(np.float64)
        aM = np.abs(Ms[d].astype(np.float64))
        y, yref = outs[d], ref_outs[d]
        ascending = (d == 0) != bptt
        order = list(range(T)) if ascending else list(range(T - 1, -1, -1))
        prev = np.zeros(y.shape[1:], np.float32)
        first = True
        tr = 0.0
        for t in order:
            live = t < lens
            yt = y[t].astype(np.float64)
            if live.any() and np.any(prev):
                xt = x_in[t]
                S = np.abs(xt) + np.abs(prev.astype(np.float64)).dot(aM)
                zr = xt + rna(prev).astype(np.float64).dot(Mr)
                zt = xt + trunc(prev).astype(np.float64).dot(Mt)
                if bptt:
                    act = acts[d][t].astype(np.float64)
                    keep = (act > 0) & (act < sg.MAXACT)
                    y64, ytr = np.where(keep, zr, 0.0), np.where(keep, zt, 0.0)
                else:
                    y64, ytr = np.clip(zr, 0.0, sg.MAXACT), np.clip(zt, 0.0, sg.MAXACT)
                Sl = S[live]
                pos = Sl > 0
                e = np.abs(yt - y64)[live]
                assert np.all(e[Sl == 0] == 0), "inexact where S = 0 (t=%d)" % t
                if pos.any():
                    worst["ratio"] = max(worst["ratio"], float(np.max(e[pos] / (U32 * Sl[pos]))))
                    et = np.abs(ytr - y64)[live]
                    tr = max(tr, float(np.max(et[pos] / (U32 * Sl[pos]))) / bound)
                    if first:
                        ef = np.abs(yref[t].astype(np.float64) - y64)[live]
                        worst["f32"] = max(worst["f32"], float(np.max(ef[pos] / (U32 * Sl[pos]))) / bound)
                        first = False
            prev = y[t]
        worst["trunc"] = min(worst["trunc"], tr)
    if worst["trunc"] == np.inf:
        worst["trunc"] = 0.0
    return worst


def _case(name, H, B, T, ndir, torch, lens="ragged", vals="clip", dmode="randn"):
    f32_plan = _raw_plan("ctcb_debug_sweep_plan", H, B, ndir)
    plan = _raw_plan("ctcb_debug_sweep_plan_tf32", H, B, ndir)
    sw = sg._problem(torch, H, B, T, ndir, 1000 * H + B + T, lens, vals, dmode)
    ref = sw.run()
    with _tf32_entry():
        r = sw.run()
        again = sw.run()
    sg._check_exact(r, sw)
    assert sg._same_run(r, again), "a rerun gave other bytes"
    rec = dict(sweep=name, H=H, B=B, T=T, ndir=ndir, plan=plan)
    if plan["kernel"] != 2:           # no TF32 mode: the fp32-faithful kernel's plan and bytes
        assert plan == f32_plan, (plan, f32_plan)
        rec["f32_bytes"] = sg._same_run(r, ref)
        print(json.dumps(rec))
        assert rec["f32_bytes"]
        return
    # the TF32 plan: the default's cluster size, splits and wgmma N; the ring of half-size stages is its own
    assert all(plan[k] == f32_plan[k] for k in ("kernel", "CS", "groups", "NP")), (plan, f32_plan)
    assert plan["stages"] >= f32_plan["stages"], (plan, f32_plan)
    bound = TF32_C0 + TF32_C1 * (H // plan["CS"] // 32)
    fwd = _steps_tf32(sw, r["F"], sw.pre, [w.T for w in sw.Ws], None, bound, ref["F"])
    # the fp32-faithful BPTT from the TF32 run's forward states, so that both see the same masks
    refb = sw.run(fwd=r)
    bptt = _steps_tf32(sw, r["dF"], sw.d, sw.Ws, r["act"], bound, refb["dF"])
    rec.update(f32_plan=f32_plan, bound=bound, fwd=fwd, bptt=bptt)
    print(json.dumps(rec))
    assert fwd["ratio"] <= bound and bptt["ratio"] <= bound, rec
    if T >= 2:
        assert min(fwd["trunc"], bptt["trunc"]) >= MARGIN, rec
        assert min(fwd["f32"], bptt["f32"]) >= MARGIN, rec


@pytest.mark.parametrize("H,B,T", [(1024, 16, 12), (1024, 128, 10), (1024, 40, 9), (1024, 3, 7), (2048, 32, 8),
                                   (2048, 256, 5), (1536, 20, 6), (1024, 200, 5), (2048, 100, 4), (512, 32, 50),
                                   (128, 8, 40)])
def test_sweep_tf32_forward_and_bptt(H, B, T, cuda):
    _case("%d-%d-%d" % (H, B, T), H, B, T, 2, cuda)


@pytest.mark.parametrize("H,B,T,ndir,forced,recipe,expect", sg.PLAN_CASES)
def test_sweep_tf32_plan(H, B, T, ndir, forced, recipe, expect, request, gknobs, cuda):
    for k, v in forced.items():
        gknobs(k, v)
    sg._check_plan(H, B, ndir, expect, cuda)
    _case(request.node.callspec.id, H, B, T, ndir, cuda, **recipe)
