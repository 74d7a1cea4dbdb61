"""GPU unit test of the dense contraction in TF32 mode (ctcb_gemm_tf32, ctcb_gemm_pair_tf32) on every case of
test_gemm_plans_gpu.py, against float64 of the operands rounded to TF32.

In TF32 mode each product on the tensor cores reads both operands rounded to the nearest TF32 value (ties away from zero;
rna below is NumPy's statement of it) and is one MMA, accumulated in fp32 (include/ctcb200.h).  With C64r = float64 of
the rounded operands and S and L as in test_gemm_plans_gpu.py, element-wise:
    |C - C64r| <= (c0 + c1 L) 2^-24 S                    (the rounded-operand bound)
    |C - C64|  <= 2 2^-11 S + (c0 + c1 L) 2^-24 S        (C64 of the unrounded operands: each rounding is <= 2^-11)
Negative controls on the same arrays must miss C64r by at least MARGIN times the rounded-operand bound somewhere: the
truncated operands' float64 product (what the MMA would read without the rounding), and ctcb_gemm_f32's result (the
3xTF32 product: if it were the one that ran, the single pass would not have).  A case whose plan is the FFMA kernel
returns ctcb_gemm_f32's bytes.  The TF32 plan keeps the default plan's BN, splits, operand paths and pair decision,
its ring stages are its own (STAGES), and every case runs twice with the same bytes.  Masked elements are exactly 0,
and C's padding and the workspace guard are untouched, as in the fp32-faithful test.  Each case prints its plan, L,
ratios and controls as one JSON line (pytest -s)."""
import ctypes
import json

import numpy as np
import pytest

import test_gemm_plans_gpu as gp
from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
# (c0, c1) of the rounded-operand bound, from the cases of this file on an H100 80GB HBM3 (power limit 700 W), by the
# rule of test_gemm_plans_gpu.py: c0 at most 4x the largest ratio |C - C64r| / (2^-24 S) measured (10.5, at L = 16), c1
# at most 4x the largest ratio / L over the chains of 32 k-blocks or more (0.123: 6.17 at L = 50).
TF32_BOUND = (40.0, 0.45)
MARGIN = 10.0              # the negative controls miss C64r by at least this many rounded-operand bounds
# Beyond this K the rounding errors of random operands (about 2^-11 |a b| each, of random sign) average out to less
# than MARGIN bounds relative to S, which grows with K: measured down to 2.4 bounds for the 3xTF32 control at K = 6400.
CONTROL_MAX_K = 4096
# ring stages of the TF32 plans: the fp32-faithful ring's shared memory in TF32 stages (K-major B: no low-half slot)
STAGES = {(64, False): 5, (64, True): 4, (128, False): 4, (128, True): 3}


def rna(x):
    """float32 -> float32 rounded to the nearest TF32 value, ties away from zero (finite x)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def trunc(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return (u & np.uint32(0xffffe000)).view(np.float32)


def _rna_t(x):
    """rna on a float32 torch tensor, on the device."""
    import torch
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xffffffff
    u = (u + 0x1000) & 0xffffe000
    return torch.where(u >= 2 ** 31, u - 2 ** 32, u).to(torch.int32).view(torch.float32)


def _trunc_t(x):
    import torch
    return (x.contiguous().view(torch.int32) & np.int32(-8192)).view(torch.float32)


def _plan_tf32(ta, tb, M, N, K, A, lda, B, ldb, problems=1):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan_tf32(ta, tb, M, N, K, A, lda, B, ldb, problems, out))
    return dict(zip(gp.FIELDS, list(out)))


def _expect_tf32(plan):
    """The TF32 plan that goes with a default plan."""
    want = dict(plan)
    if plan["kernel"] == 1:
        want["stages"] = STAGES[(plan["BN"], plan["b_path"] == gp.MN)]
    return want


def _run_tf32(call):
    """call.run with ctcb_gemm_tf32."""
    import _ctcb
    from _ctcb import lib, check, ptr
    c = call.c
    if call.C.numel():
        call.C.copy_(gp._torch().from_numpy(call.c0).cuda())
    check(lib.ctcb_gemm_tf32(c["ta"], c["tb"], c["M"], c["N"], c["K"], call.alpha, call.a_ptr, call.lda, call.b_ptr,
                             call.ldb, call.beta, call.C.data_ptr(), call.ldc, ptr(call.bias), call.relu,
                             None if call.mask is None else call.mask.data_ptr(), ptr(call.ws), call.ws_bytes,
                             _ctcb.current_stream()))
    gp._torch().cuda.synchronize()
    return call.C.cpu().numpy()


def _reference_of(call, fn):
    """Call.reference() of the operands mapped through fn (rna, trunc, or None for the operands themselves)."""
    if fn is None:
        return call.reference()
    a, b = call.a_op, call.b_op
    call.a_op, call.b_op = fn(a), fn(b)
    try:
        return call.reference()
    finally:
        call.a_op, call.b_op = a, b


def _ratio(got, want, S, keep):
    diff = np.abs(got.astype(np.float64) - want)
    r = np.where(S > 0, diff / np.maximum(U * S, 1e-300), np.where(diff > 0, np.inf, 0.0))
    return float(r[keep].max()) if keep.any() else 0.0


def _tf32_record(got, call, L, f32_out):
    """Ratios of the TF32 result and of both controls; the bound checks of this file."""
    c0, c1 = TF32_BOUND
    bound = c0 + c1 * L
    keep = np.ones(got.shape, bool) if call.mask_np is None else (call.mask_np > 0)
    want_r, S = _reference_of(call, _rna_t)
    want, _ = _reference_of(call, None)
    want_t, _ = _reference_of(call, _trunc_t)
    rec = dict(L=L, bound=bound, ratio=_ratio(got, want_r, S, keep),
               ratio_unrounded=_ratio(got, want, S, keep), finite=bool(np.isfinite(got).all()),
               trunc_control=_ratio(want_t.astype(np.float32), want_r, S, keep) / bound,
               f32_control=_ratio(f32_out, want_r, S, keep) / bound)
    rec["within"] = rec["ratio"] <= bound
    rec["within_unrounded"] = rec["ratio_unrounded"] <= 2 * 2.0 ** 13 + bound
    if call.mask_np is not None:
        rec["masked_zero"] = bool((got[~keep] == 0).all())
    return rec


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", list(gp.CASES))
def test_gemm_tf32_plan(name, knobs, cuda):
    c = gp.CASES[name]
    cuda.cuda.empty_cache()
    if c.get("simt"):
        knobs("CTCB_GEMM", "simt")
    if c.get("tc_copy"):
        knobs("CTCB_GEMM_TC_COPY", "1")
    call = gp.Call(name, c)
    plan = call.plan()
    gp._check_plan(plan, c["plan"], name)
    tplan = _plan_tf32(c["ta"], c["tb"], c["M"], c["N"], c["K"], call.a_ptr, call.lda, call.b_ptr, call.ldb)
    assert tplan == _expect_tf32(plan), (tplan, plan)
    got = _run_tf32(call)
    again = _run_tf32(call)
    same = np.array_equal(got.view(np.uint32), again.view(np.uint32))
    ok_c, ok_ws = call.untouched()
    f32 = call.run()
    if plan["kernel"] == 0:           # the FFMA kernel: ctcb_gemm_f32's bytes
        rec = dict(plan=tplan, same_bytes=same, f32_bytes=bool(np.array_equal(got.view(np.uint32), f32.view(np.uint32))))
        print(json.dumps({"gemm_tf32_" + name: rec}))
        assert same and ok_c and ok_ws and rec["f32_bytes"], rec
        return
    call.ws = None
    rec = _tf32_record(got, call, gp._chain(tplan, c["K"]), f32)
    rec.update(plan=tplan, same_bytes=same, c_untouched=ok_c, guard_untouched=ok_ws)
    print(json.dumps({"gemm_tf32_" + name: rec}))
    assert same and ok_c and ok_ws, rec
    assert rec["finite"] and rec.get("masked_zero", True), rec
    assert rec["within"] and rec["within_unrounded"], rec
    if c["K"] <= CONTROL_MAX_K:
        assert rec["trunc_control"] >= MARGIN and rec["f32_control"] >= MARGIN, rec


@pytest.mark.parametrize("name", list(gp.PAIRS))
def test_gemm_pair_tf32(name, cuda):
    """The pair in TF32 mode: each result has the bytes of its single ctcb_gemm_tf32 call and meets the bound."""
    import _ctcb
    from _ctcb import lib, check, ptr
    import zlib
    torch = cuda
    H, K, alpha, beta, a1_off, room, expect = gp.PAIRS[name]
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))
    ops = [torch.randn(K * H + 8, device="cuda", generator=gen) for _ in range(4)]
    A = [ops[0][:K * H].view(K, H), ops[1][a1_off:a1_off + K * H].view(K, H)]
    B = [ops[2][:K * H].view(K, H), ops[3][:K * H].view(K, H)]
    c0 = torch.randn(2, H, H, device="cuda", generator=gen)
    single_ws = lib.ctcb_gemm_workspace_bytes(H, H, K)
    ws_bytes = lib.ctcb_gemm_pair_workspace_bytes(H, H, K) if room == "pair" else single_ws
    ws = torch.full((ws_bytes + gp.GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    plan = gp._plan(1, 0, H, H, K, A[1].data_ptr(), H, B[1].data_ptr(), H, problems=2)
    gp._check_plan(plan, expect, name)
    tplan = _plan_tf32(1, 0, H, H, K, A[1].data_ptr(), H, B[1].data_ptr(), H, problems=2)
    assert tplan == _expect_tf32(plan), (tplan, plan)
    st = _ctcb.current_stream()
    C = c0.clone()
    check(lib.ctcb_gemm_pair_tf32(1, 0, H, H, K, alpha, A[0].data_ptr(), A[1].data_ptr(), H, B[0].data_ptr(),
                                  B[1].data_ptr(), H, beta, ptr(C[0]), ptr(C[1]), H, ptr(ws), ws_bytes, st))
    torch.cuda.synchronize()
    guard = bool((ws[ws_bytes:] == 0xA5).all())
    S1, F = c0.clone(), c0.clone()
    wss = torch.empty(single_ws, dtype=torch.uint8, device="cuda")
    for q in range(2):
        check(lib.ctcb_gemm_tf32(1, 0, H, H, K, alpha, A[q].data_ptr(), H, B[q].data_ptr(), H, beta, ptr(S1[q]), H,
                                 None, 0, None, ptr(wss), single_ws, st))
        check(lib.ctcb_gemm_f32(1, 0, H, H, K, alpha, A[q].data_ptr(), H, B[q].data_ptr(), H, beta, ptr(F[q]), H,
                                None, 0, None, ptr(wss), single_ws, st))
    torch.cuda.synchronize()
    same = bool(torch.equal(C.view(torch.int32), S1.view(torch.int32)))
    recs = []
    for q in range(2):
        qplan = _plan_tf32(1, 0, H, H, K, A[q].data_ptr(), H, B[q].data_ptr(), H)
        got = C[q].cpu().numpy()
        if qplan["kernel"] == 0:
            recs.append(dict(plan=qplan, f32_bytes=bool(torch.equal(C[q].view(torch.int32), F[q].view(torch.int32)))))
            continue
        L = gp._chain(qplan, K)
        bound = TF32_BOUND[0] + TF32_BOUND[1] * L
        c0q = c0[q].cpu().numpy().astype(np.float64)
        P, S = gp._product(_rna_t(A[q].T), _rna_t(B[q]))
        want_r = alpha * P + beta * c0q
        S = abs(alpha) * S + abs(beta) * np.abs(c0q)
        P0, _ = gp._product(A[q].T, B[q])
        Pt, _ = gp._product(_trunc_t(A[q].T), _trunc_t(B[q]))
        keep = np.ones(got.shape, bool)
        recs.append(dict(L=L, bound=bound, ratio=_ratio(got, want_r, S, keep),
                         ratio_unrounded=_ratio(got, alpha * P0 + beta * c0q, S, keep),
                         trunc_control=_ratio((alpha * Pt + beta * c0q).astype(np.float32), want_r, S, keep) / bound,
                         f32_control=_ratio(F[q].cpu().numpy(), want_r, S, keep) / bound))
    print(json.dumps({"gemm_pair_tf32_" + name: dict(plan=tplan, same_bytes=same, guard_untouched=guard,
                                                     problems=recs)}))
    assert same and guard
    for r in recs:
        if "f32_bytes" in r:
            assert r["f32_bytes"], r
            continue
        assert r["ratio"] <= r["bound"] and r["ratio_unrounded"] <= 2 * 2.0 ** 13 + r["bound"], r
        if K <= CONTROL_MAX_K:
            assert r["trunc_control"] >= MARGIN and r["f32_control"] >= MARGIN, r
