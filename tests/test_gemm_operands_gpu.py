"""GPU test of how the tensor-core contraction (gemm_tc.cu) reads its operands.

wgmma reads .tf32 operands K-major only.  An operand stored MN-major (A as [K][M], B as [K][N]: every weight gradient
over the time-major activations) is read in place and transposed in shared memory; an operand TMA cannot describe
(pitch not a multiple of 16 bytes, base not 16-byte aligned) is copied into the workspace first.  Every case checks its
plan with ctcb_debug_gemm_plan (operand paths, splits, accumulator chains of at most 64 k-blocks), its
result against a float64 product, and, with CTCB_GEMM_TC_COPY=1 set in process, that the copy path gives the same
bytes at the same split.  The recurrent weight-gradient pair (one launch for both directions) must equal two single
calls byte for byte.  Each case prints its plan and error as one JSON line (shown with pytest -s)."""
import json
import zlib

import numpy as np
import pytest

from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
H100_SMS = 132             # the split counts below are those of the 132-SM H100 SXM
CHAIN_KB = 64              # TC_CHAIN_KB: k-blocks of 32 per accumulator chain
# Frobenius-relative error against float64.  The tensor-core accumulator truncates, so the error of 3xTF32 grows with
# the k-blocks each accumulator chain adds up (kb_per_split): measured on an H100 80GB HBM3 (power limit 400 W) 2.1e-6 at
# 8 k-blocks and 1.2e-5 at 50.  The bound is BOUND_FIXED + BOUND_PER_KB * kb_per_split.
BOUND_FIXED, BOUND_PER_KB = 2e-6, 4e-7
KMAJOR, MN, COPY = 0, 1, 2
B_C2, H_C2, T_C2 = 32, 512, 200
R_C2 = B_C2 * T_C2

# name: (transA, transB, M, N, K, beta, {extra}, expected (A path, B path, splits on 132 SMs))
#   extra: lda / ldb pitch padding (elements), a_off / b_off (elements from a 16-byte aligned base)
CASES = {
    # the contractions of the C2 step (H = 512, B = 32, T = 200)
    "c2_dW3": (1, 0, 62, 512, R_C2, 0.0, {}, (COPY, MN, 25)),        # delta3 has a 248-byte row pitch
    "c2_dW2": (1, 0, 512, 512, R_C2, 0.0, {}, (MN, MN, 9)),
    "c2_delta1": (0, 0, R_C2, 512, 512, 0.0, {}, (KMAJOR, MN, 1)),
    "c2_dW1": (1, 0, 512, 41, R_C2, 0.0, {}, (MN, COPY, 25)),         # feats has a 164-byte row pitch
    "c2_dW2_beta1": (1, 0, 512, 512, R_C2, 1.0, {}, (MN, MN, 9)),
    # every orientation, ragged M / N / K
    "t00_ragged": (0, 0, 260, 40, 200, 0.0, {}, (KMAJOR, MN, 1)),
    "t01_ragged": (0, 1, 300, 200, 1000, 0.0, {}, (KMAJOR, KMAJOR, 4)),
    "t10_ragged": (1, 0, 200, 72, 300, 0.0, {}, (MN, MN, 1)),
    "t11_ragged": (1, 1, 256, 96, 520, 1.0, {}, (MN, KMAJOR, 2)),
    "t10_three_splits": (1, 0, 1024, 768, 1024, 0.0, {}, (MN, MN, 3)),
    "t00_chain_bound": (0, 0, 1024, 1024, 6400, 0.0, {}, (KMAJOR, MN, 4)),
    # layouts TMA cannot describe fall back to the copy
    "t10_odd_pitch": (1, 0, 192, 256, 2000, 0.0, {"lda": 1}, (COPY, MN, 7)),
    "t00_unaligned_base": (0, 0, 384, 128, 700, 1.0, {"b_off": 1}, (KMAJOR, COPY, 2)),
}


def _dev():
    import torch
    return torch


def _operand(rng, rows, cols, pad, off):
    """rows x cols float32 with pitch cols + pad, starting `off` floats into its allocation; (numpy, tensor, view, ld)."""
    torch = _dev()
    ld = cols + pad
    x = rng.randn(rows, cols).astype(np.float32)
    buf = torch.zeros(off + rows * ld + 4, dtype=torch.float32, device="cuda")
    view = buf[off:off + rows * ld].view(rows, ld)
    view[:, :cols].copy_(torch.from_numpy(x))
    return x, buf, view, ld


def _plan(ta, tb, M, N, K, A, lda, Bp, ldb, problems=1):
    from _ctcb import lib, check
    import ctypes
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan(ta, tb, M, N, K, A, lda, Bp, ldb, problems, out))
    return dict(zip(("kernel", "BN", "stages", "splits", "ctas", "a_path", "b_path", "problems"), list(out)))


def _run_case(name):
    """Result (numpy float32), plan and float64 reference of one case, computed on the plan of the knobs in effect."""
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = _dev()
    ta, tb, M, N, K, beta, ex, _ = CASES[name]
    rng = np.random.RandomState(zlib.crc32(name.encode()))
    a, abuf, A, lda = _operand(rng, *((K, M) if ta else (M, K)), ex.get("lda", 0), ex.get("a_off", 0))
    b, bbuf, Bm, ldb = _operand(rng, *((K, N) if not tb else (N, K)), ex.get("ldb", 0), ex.get("b_off", 0))
    c0 = rng.randn(M, N).astype(np.float32)
    C = torch.from_numpy(c0).cuda()
    ws = torch.empty(lib.ctcb_gemm_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    plan = _plan(ta, tb, M, N, K, A.data_ptr(), lda, Bm.data_ptr(), ldb)
    check(lib.ctcb_gemm_f32(ta, tb, M, N, K, 1.0, A.data_ptr(), lda, Bm.data_ptr(), ldb, beta, ptr(C), N, None, 0, None,
                            ptr(ws), ws.numel(), _ctcb.current_stream()))
    torch.cuda.synchronize()
    a64 = a.astype(np.float64).T if ta else a.astype(np.float64)
    b64 = b.astype(np.float64) if not tb else b.astype(np.float64).T
    want = a64 @ b64 + beta * c0.astype(np.float64)
    return C.cpu().numpy(), plan, want


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def _sms():
    return _dev().cuda.get_device_properties(0).multi_processor_count


def _bound(plan, K):
    nkb = (K + 31) // 32
    kb_per_split = (nkb + plan["splits"] - 1) // plan["splits"]
    return BOUND_FIXED + BOUND_PER_KB * kb_per_split


def _check_chain(plan, M, N, K):
    """Every accumulator chain within CHAIN_KB k-blocks, and the CTA count the plan's tiles and splits make."""
    nkb = (K + 31) // 32
    assert (nkb + plan["splits"] - 1) // plan["splits"] <= CHAIN_KB, plan
    tiles = -(-M // 128) * -(-N // plan["BN"])
    assert plan["ctas"] == plan["problems"] * tiles * plan["splits"], plan


@pytest.mark.parametrize("name", list(CASES))
def test_gemm_operand_paths(name, cuda):
    ta, tb, M, N, K, beta, ex, (pa, pb, splits) = CASES[name]
    got, plan, want = _run_case(name)
    err = _rel(got, want)
    bound = _bound(plan, K)
    print(json.dumps({"gemm_" + name: dict(plan=plan, err=err, bound=bound)}))
    assert plan["kernel"] == 1 and plan["problems"] == 1
    assert (plan["a_path"], plan["b_path"]) == (pa, pb), plan
    if _sms() == H100_SMS:
        assert plan["splits"] == splits, plan
    _check_chain(plan, M, N, K)
    assert np.isfinite(got).all()
    assert err < bound, (err, bound)


def test_gemm_copy_path_same_bytes(knobs, cuda):
    """CTCB_GEMM_TC_COPY=1: the same cases through the workspace copies, byte for byte."""
    in_place = {name: _run_case(name)[:2] for name in CASES}
    knobs("CTCB_GEMM_TC_COPY", "1")
    for name in CASES:
        ref, ref_plan, _ = _run_case(name)
        got, plan = in_place[name]
        splits, a_path, b_path = ref_plan["splits"], ref_plan["a_path"], ref_plan["b_path"]
        assert splits == plan["splits"], (name, splits, plan)
        # the copy path reads nothing MN-major in place
        assert a_path != MN and b_path != MN, name
        assert (a_path, b_path) == tuple(COPY if p == MN else p for p in (plan["a_path"], plan["b_path"])), name
        same = np.array_equal(got.view(np.uint32), ref.view(np.uint32))
        print(json.dumps({"gemm_copy_" + name: dict(splits=splits, same_bytes=same)}))
        assert same, name


def _pair_inputs(H, R, seed):
    """Time-major buffers as the BPTT sweep leaves them: dFor, For, dBack, Back, each [T][B][H] = R x H."""
    torch = _dev()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(R, H, device="cuda", generator=g) for _ in range(4)]


@pytest.mark.parametrize("H,B,T,beta", [(512, 32, 200, 0.0), (512, 32, 200, 1.0), (1024, 32, 201, 0.0), (256, 16, 20, 1.0)])
def test_gemm_recurrent_pair(H, B, T, beta, cuda):
    """dWtf = dFor[B:]^T For[:-B] and dWtb = dBack[:-B]^T Back[B:] in one launch: against float64, and against two
    single calls byte for byte (the pair keeps the single call's split)."""
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    R = T * B
    Rm = R - B
    dF, F, dB, Bk = _pair_inputs(H, R, seed=H + T)
    A0, B0 = dF[B:], F[:Rm]             # dFor + B*H, For
    A1, B1 = dB[:Rm], Bk[B:]            # dBack, Back + B*H
    c0 = torch.randn(2, H, H, device="cuda")
    C = c0.clone()
    st = _ctcb.current_stream()
    ws = torch.empty(lib.ctcb_gemm_pair_workspace_bytes(H, H, Rm), dtype=torch.uint8, device="cuda")
    plan = _plan(1, 0, H, H, Rm, A0.data_ptr(), H, B0.data_ptr(), H, problems=2)
    single = _plan(1, 0, H, H, Rm, A0.data_ptr(), H, B0.data_ptr(), H, problems=1)
    check(lib.ctcb_gemm_pair_f32(1, 0, H, H, Rm, 1.0, A0.data_ptr(), A1.data_ptr(), H, B0.data_ptr(), B1.data_ptr(), H,
                                 beta, ptr(C[0]), ptr(C[1]), H, ptr(ws), ws.numel(), st))
    torch.cuda.synchronize()
    errs = []
    for q, (Aq, Bq) in enumerate(((A0, B0), (A1, B1))):
        want = Aq.double().T @ Bq.double() + beta * c0[q].double()
        errs.append(_rel(C[q].cpu().numpy(), want.cpu().numpy()))
    rec = dict(plan=plan, single_splits=single["splits"], err=errs, bound=_bound(plan, Rm))
    assert plan["problems"] == 2 and (plan["a_path"], plan["b_path"]) == (MN, MN), plan
    _check_chain(plan, H, H, Rm)
    assert max(errs) < _bound(plan, Rm), (errs, _bound(plan, Rm))
    assert single["splits"] == plan["splits"], (single, plan)
    S = c0.clone()
    wss = torch.empty(lib.ctcb_gemm_workspace_bytes(H, H, Rm), dtype=torch.uint8, device="cuda")
    for q, (Aq, Bq) in enumerate(((A0, B0), (A1, B1))):
        check(lib.ctcb_gemm_f32(1, 0, H, H, Rm, 1.0, Aq.data_ptr(), H, Bq.data_ptr(), H, beta, ptr(S[q]), H, None, 0,
                                None, ptr(wss), wss.numel(), st))
    torch.cuda.synchronize()
    rec["same_bytes"] = bool(torch.equal(S.view(torch.int32), C.view(torch.int32)))
    assert rec["same_bytes"]
    print(json.dumps({"gemm_pair_%d_%d_%d_b%d" % (H, B, T, int(beta)): rec}))
