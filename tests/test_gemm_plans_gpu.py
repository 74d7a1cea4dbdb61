"""GPU unit test of the dense contraction (ctcb_gemm_f32, ctcb_gemm_pair_f32) on every plan its planners can choose,
against a float64 product with element-wise bounds.

Two kernels run a contraction: the exact-fp32 FFMA kernel (gemm_simt.cu; K < 128, M < 32, N < 32, a short workspace, or
CTCB_GEMM=simt) and the 3xTF32 tensor-core kernel (gemm_tc.cu).  Their plans differ in output tile width and ring
stages, K splits (a split-K reduce then runs the epilogue), how each operand is read (16-byte loads or not; K-major or
MN-major in place, or copied into the workspace first) and whether a pair shares one launch.  Every case names the plan
it targets and checks it with ctcb_debug_gemm_plan before launching; knobs are set in process (recipes.knobs) before any
workspace is sized.  On a device that is not a 132-SM H100 a case whose plan is out of reach skips.

Reference: C64 = alpha op(A) op(B) + beta C0 + bias in float64, then ReLU and the mask, and S = |alpha| |op(A)| |op(B)| +
|beta C0| + |bias|.  Element-wise, |C - C64| <= (c0 + c1 L) 2^-24 S, where L is the length of the plan's accumulator
chains: k per split for the FFMA kernel, k-blocks of 32 per split for the tensor cores.  Masked elements are exactly 0;
the mask carries 0, -0.0, a positive denormal, negatives and positives, and "masked" means not (mask > 0) as NumPy says.
Every call gets exactly the workspace ctcb_gemm_workspace_bytes reports, followed by a guard, and C a row pitch ldc and
rows after it: guard, padding and trailing rows are filled with a sentinel and must come back unchanged.  Every case
runs twice and must give the same bytes.  Each case prints its plan, L, error ratio and bound as one JSON line (shown
with pytest -s)."""
import ctypes
import json
import zlib

import numpy as np
import pytest

from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
H100_SMS = 132             # the split counts below are those of the 132-SM H100 SXM
FIELDS = ("kernel", "BN", "stages", "splits", "ctas", "a_path", "b_path", "problems")
U = 2.0 ** -24
# (c0, c1) per kernel, from the cases of this file on an H100 80GB HBM3 (power limit 400 W; DESIGN.md section 4): c0 at
# most 4x the largest ratio |C - C64| / (2^-24 S) measured, c1 at most 4x the largest ratio / L over the chains of 32 k
# or more (k-blocks for the tensor cores).  FFMA (round-to-nearest fp32 chains, then the split sum and the epilogue):
# 5.30 and 0.127.  Tensor cores (3xTF32: lo.lo dropped, lo read as TF32, a truncating accumulator): 30.2 and 0.391.
BOUNDS = {0: (21.0, 0.5), 1: (120.0, 1.5)}
SENTINEL = 7.0
GUARD = 4096               # bytes of 0xA5 after the workspace
KMAJOR, MN, COPY = 0, 1, 2
SMALL = 1 << 26            # M N K up to this: the float64 reference on the host (NumPy), above it on the device
GEMM_MAX_M = 128 * 65535


def F(splits, vec):
    return dict(kernel=0, BN=128, splits=splits, a_path=vec, b_path=0, problems=1)


def T(BN, splits, a_path, b_path, problems=1):
    return dict(kernel=1, BN=BN, stages=4 if BN == 64 else 3, splits=splits, a_path=a_path, b_path=b_path,
                problems=problems)


def case(ta, tb, M, N, K, plan, **kw):
    return dict(ta=ta, tb=tb, M=M, N=N, K=K, plan=plan, **kw)


EPILOGUES = {
    "none": {},
    "bias": dict(bias=True),
    "bias_relu": dict(bias=True, relu=True),
    "mask": dict(mask=True),
    "beta1": dict(beta=1.0),
    "beta0_nan": dict(nan_c0=True),                       # beta = 0 must not read C0
    "alpha": dict(alpha=-0.5, beta=1.0, bias=True),
    "ldc_n3": dict(ldc_pad=3, beta=1.0, bias=True, mask=True),
}
# one shape per kernel and store path: (ta, tb, M, N, K, plan)
EPI_SHAPES = {
    "ffma_direct": (0, 1, 300, 200, 100, F(1, 1)),
    "ffma_reduce": (1, 0, 20, 300, 5000, F(35, 1)),
    "tc_direct": (0, 1, 300, 200, 400, T(128, 1, KMAJOR, KMAJOR)),
    "tc_reduce": (1, 0, 300, 200, 3000, T(128, 11, MN, MN)),
}

CASES = {}
# ---- FFMA: four orientations x 16-byte loads on / off (odd pitch of A, B one float off its aligned base), K ragged
for ta in (0, 1):
    for tb in (0, 1):
        o = "%d%d" % (ta, tb)
        CASES["f%s_vec" % o] = case(ta, tb, 200, 150, 97, F(1, 1), ldc_pad=2, bias=True, relu=True, beta=1.0)
        CASES["f%s_odd_pitch" % o] = case(ta, tb, 200, 150, 97, F(1, 0), a_pad=ta, ldc_pad=2, bias=True, beta=1.0)
        CASES["f%s_base_off" % o] = case(ta, tb, 200, 150, 97, F(1, 0), b_off=1, ldc_pad=2, mask=True)
# float4 epilogue (ldc % 4 == 0, C and mask 16-byte aligned) and each thing that turns it off
CASES["f_vecc_on"] = case(0, 1, 200, 150, 97, F(1, 1), ldc_pad=2, bias=True, mask=True, beta=1.0)
CASES["f_vecc_odd_ldc"] = case(0, 1, 200, 150, 97, F(1, 1), ldc_pad=3, bias=True, mask=True, beta=1.0)
CASES["f_vecc_c_off"] = case(0, 1, 200, 150, 97, F(1, 1), ldc_pad=2, c_off=1, bias=True, mask=True, beta=1.0)
CASES["f_vecc_mask_off"] = case(0, 1, 200, 150, 97, F(1, 1), ldc_pad=2, m_off=1, bias=True, mask=True, beta=1.0)
# split-K (M < 32): float4 partials (N % 4 == 0) and scalar ones
CASES["f_split_n300"] = case(1, 0, 20, 300, 5000, F(35, 1), bias=True, relu=True)
CASES["f_split_n301"] = case(1, 0, 20, 301, 5000, F(35, 1), beta=1.0, mask=True)
CASES["f_split_n301_novec"] = case(1, 0, 20, 301, 5000, F(35, 0), b_pad=0, beta=1.0)
# forced at tensor-core shapes
CASES["f_simt_t10_split"] = case(1, 0, 1000, 512, 3000, F(9, 1), simt=True, beta=1.0)
CASES["f_simt_t01_wide"] = case(0, 1, 6400, 512, 512, F(1, 1), simt=True, bias=True, relu=True)
CASES["f_simt_t00_ragged"] = case(0, 0, 333, 257, 1001, F(7, 0), simt=True, a_pad=0, mask=True)
CASES["f_simt_t11_ragged"] = case(1, 1, 333, 257, 1001, F(7, 1), simt=True, alpha=-0.5, bias=True)
# degenerate sizes
CASES["f_k0"] = case(0, 1, 50, 40, 0, F(1, 1), a_pad=4, b_pad=4, beta=1.0, bias=True, relu=True)
CASES["f_k0_mask"] = case(0, 0, 50, 40, 0, F(1, 1), a_pad=4, alpha=-0.5, beta=0.5, mask=True)
CASES["f_m0"] = case(0, 1, 0, 40, 10, dict(kernel=0, splits=0), beta=1.0, bias=True)
CASES["f_n0"] = case(0, 1, 30, 0, 10, dict(kernel=0, splits=0), beta=1.0)
CASES["f_1x1x1"] = case(0, 0, 1, 1, 1, F(1, 0), a_pad=0, b_pad=0, beta=1.0, bias=True)
# ---- tensor cores: tile widths, the four in-place operand layouts, the copies, split counts
CASES["t01_bn64_n48"] = case(0, 1, 300, 48, 400, T(64, 1, KMAJOR, KMAJOR), bias=True)
CASES["t10_bn64_n64"] = case(1, 0, 300, 64, 400, T(64, 1, MN, MN), beta=1.0)
CASES["t00_bn128_n65"] = case(0, 0, 300, 65, 400, T(128, 1, KMAJOR, MN), mask=True)
CASES["t11_bn128_n129"] = case(1, 1, 300, 129, 400, T(128, 1, MN, KMAJOR), bias=True, relu=True)
CASES["t01_bn128_n512"] = case(0, 1, 300, 512, 400, T(128, 1, KMAJOR, KMAJOR))
CASES["t10_copy_knob"] = case(1, 0, 300, 200, 3000, T(128, 11, COPY, COPY), tc_copy=True, bias=True)
CASES["t01_copy_k3001"] = case(0, 1, 300, 200, 3001, T(128, 11, COPY, COPY), a_pad=0, b_pad=0, beta=1.0)
CASES["t00_copy_a_off"] = case(0, 0, 300, 200, 3000, T(128, 11, COPY, MN), a_off=1, mask=True)
CASES["t10_copy_odd_lda"] = case(1, 0, 300, 200, 3000, T(128, 11, COPY, MN), a_pad=1, beta=1.0)
CASES["t10_copy_both_odd"] = case(1, 0, 300, 200, 3000, T(128, 11, COPY, COPY), a_pad=1, b_pad=1, bias=True)
CASES["t01_fill16"] = case(0, 1, 256, 256, 4096, T(128, 16, KMAJOR, KMAJOR), bias=True)
CASES["t11_k1000"] = case(1, 1, 200, 100, 1000, T(128, 4, MN, KMAJOR), beta=1.0)
CASES["t01_m40"] = case(0, 1, 40, 200, 600, T(128, 2, KMAJOR, KMAJOR), mask=True)
CASES["t01_chain33_one_tile"] = case(0, 1, 128, 64, 67000, T(64, 33, KMAJOR, KMAJOR), bias=True)
CASES["t10_chain33_1536"] = case(1, 0, 1536, 1536, 67000, T(128, 33, MN, MN))
# ---- every epilogue on both kernels, on the direct store and in the split-K reduce
for sname, (ta, tb, M, N, K, plan) in EPI_SHAPES.items():
    for ename, ex in EPILOGUES.items():
        CASES["epi_%s_%s" % (sname, ename)] = case(ta, tb, M, N, K, plan, **ex)
# ---- the step's contractions (DESIGN.md section 2) at C2 (D 41, H 512, K 62) and C3 / C4 widths, at its pitches
for R, tag in ((6400, "r6400"), (256, "r256")):
    big = R == 6400
    CASES["c2_fwd1_" + tag] = case(0, 1, R, 512, 41, F(1, 0), a_pad=0, b_pad=0, bias=True, relu=True)
    CASES["c2_fwd2_" + tag] = case(0, 1, R, 512, 512, T(128, 1 if big else 2, KMAJOR, KMAJOR), bias=True, relu=True)
    CASES["c2_fwd_temporal_" + tag] = case(0, 1, R, 512, 512, T(128, 1 if big else 2, KMAJOR, KMAJOR), bias=True)
    CASES["c2_logits_" + tag] = case(0, 1, R, 62, 512, T(64, 2, KMAJOR, KMAJOR), b_pad=0, bias=True)
    CASES["c2_delta_out_" + tag] = case(0, 0, R, 512, 62, F(1, 0), a_pad=0, mask=True)
    CASES["c2_delta2_" + tag] = case(0, 0, R, 512, 512, T(128, 1 if big else 2, KMAJOR, MN), mask=True)
for beta in (0.0, 1.0):
    b = "_b%d" % beta
    CASES["c2_dW_out" + b] = case(1, 0, 62, 512, 6400, T(128, 25, COPY, MN), a_pad=0, beta=beta)
    CASES["c2_dW2" + b] = case(1, 0, 512, 512, 6400, T(128, 9, MN, MN), beta=beta)
    CASES["c2_dW1" + b] = case(1, 0, 512, 41, 6400, T(64, 25, MN, COPY), b_pad=0, beta=beta)
CASES["c3_dW2_r6400"] = case(1, 0, 1024, 1024, 6400, T(128, 4, MN, MN), beta=1.0)
CASES["c4_fwd_r512"] = case(0, 1, 512, 2048, 2048, T(128, 3, KMAJOR, KMAJOR), bias=True, relu=True)
CASES["c4_delta_r512"] = case(0, 0, 512, 2048, 2048, T(128, 3, KMAJOR, MN), mask=True)
CASES["c4_dW_r512"] = case(1, 0, 2048, 2048, 512, T(128, 1, MN, MN), beta=1.0)
# ---- launch limits: a transposed copy with K beyond 65,535 tiles of 32 rows, and M at 65,535 row tiles
CASES["t10_copy_k2100000"] = case(1, 0, 62, 41, 2100000, T(64, 1026, COPY, COPY), a_pad=0, b_pad=0)
CASES["f_m_limit"] = case(0, 1, GEMM_MAX_M, 1, 1, F(1, 0), a_pad=0, b_pad=0, bias=True)


# ------------------------------------------------------------------------------------------------ helpers
def _torch():
    import torch
    return torch


def _plan(ta, tb, M, N, K, A, lda, B, ldb, problems=1):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan(ta, tb, M, N, K, A, lda, B, ldb, problems, out))
    return dict(zip(FIELDS, list(out)))


def _check_plan(plan, expect, what):
    wrong = {k: (v, plan.get(k)) for k, v in expect.items() if plan.get(k) != v}
    if wrong:
        msg = "%s: planned %s, this case targets %s" % (what, plan, expect)
        if _torch().cuda.get_device_properties(0).multi_processor_count != H100_SMS:
            pytest.skip("plan not reachable on this device: " + msg)
        pytest.fail(msg)


def _chain(plan, K):
    """L: the length of the plan's accumulator chains (k per split for FFMA, k-blocks per split for the tensor cores)."""
    if K == 0 or plan["splits"] == 0:
        return 0
    if plan["kernel"] == 0:
        kps = -(-K // plan["splits"])
        return min(K, -(-kps // 16) * 16)
    nkb = -(-K // 32)
    return -(-nkb // plan["splits"])


def _check_ctas(plan, M, N):
    if M > 0 and N > 0:
        bm, bn = 128, plan["BN"]
        assert plan["ctas"] == plan["problems"] * -(-M // bm) * -(-N // bn) * plan["splits"], plan


def _operand(gen, rows, cols, pad, off):
    """rows x cols float32 randn with pitch cols + pad, `off` floats into its allocation: (buffer, view, address, ld).
    The address is taken from the allocation, so an empty operand (K = 0) still passes a valid pointer."""
    torch = _torch()
    ld = cols + pad
    buf = torch.zeros(off + rows * ld + 4, dtype=torch.float32, device="cuda")
    view = buf[off:off + rows * ld].view(rows, ld)
    if rows * cols:
        view[:, :cols] = torch.randn(rows, cols, device="cuda", generator=gen)
    return buf, view, buf.data_ptr() + 4 * off, ld


def _mask_values(rng, M, N):
    """0, -0.0, the smallest positive denormal, negatives and positives, in random places."""
    x = rng.randn(M, N).astype(np.float32)
    kind = rng.randint(0, 5, size=(M, N))
    x[kind == 0] = 0.0
    x[kind == 1] = -0.0
    x[kind == 2] = np.float32(1.4e-45)
    x[kind == 3] = -np.abs(x[kind == 3])
    x[kind == 4] = np.abs(x[kind == 4]) + np.float32(1e-3)
    return x


def _product(a_op, b_op):
    """float64 op(A) op(B) and |op(A)| |op(B)| of float32 device views a_op (M x K) and b_op (K x N), as NumPy."""
    torch = _torch()
    M, K = a_op.shape
    N = b_op.shape[1]
    if M * N * K <= SMALL:
        a = a_op.cpu().numpy().astype(np.float64)
        b = b_op.cpu().numpy().astype(np.float64)
        return a @ b, np.abs(a) @ np.abs(b)
    P = torch.zeros(M, N, dtype=torch.float64, device="cuda")
    S = torch.zeros(M, N, dtype=torch.float64, device="cuda")
    step = max(32, (1 << 24) // (M + N))          # chunks of K: about 128 MB of float64 operands at a time
    for k0 in range(0, K, step):
        a = a_op[:, k0:k0 + step].double()
        b = b_op[k0:k0 + step].double()
        P += a @ b
        S += a.abs() @ b.abs()
        del a, b
    return P.cpu().numpy(), S.cpu().numpy()


class Call:
    """One contraction's buffers: operands, C inside a sentinel-filled buffer of pitch ldc, mask, bias, workspace."""

    def __init__(self, name, c, ws_bytes=None):
        torch = _torch()
        from _ctcb import lib
        self.c = c
        ta, tb, M, N, K = c["ta"], c["tb"], c["M"], c["N"], c["K"]
        gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))
        rng = np.random.RandomState(zlib.crc32(name.encode()) & 0x7fffffff)
        ar, ac = (K, M) if ta else (M, K)
        br, bc = (N, K) if tb else (K, N)
        apad = c.get("a_pad", (-ac) % 4)
        bpad = c.get("b_pad", (-bc) % 4)
        self.abuf, self.A, self.a_ptr, self.lda = _operand(gen, ar, ac, apad, c.get("a_off", 0))
        self.bbuf, self.B, self.b_ptr, self.ldb = _operand(gen, br, bc, bpad, c.get("b_off", 0))
        self.a_op = self.A[:, :ac].T if ta else self.A[:, :ac]
        self.b_op = self.B[:, :bc].T if tb else self.B[:, :bc]
        self.ldc = N + c.get("ldc_pad", 0)
        coff = c.get("c_off", 0)
        self.cbuf = torch.full((coff + (M + 2) * self.ldc + 8,), SENTINEL, dtype=torch.float32, device="cuda")
        self.C = self.cbuf[coff:coff + M * self.ldc].view(M, self.ldc)[:, :N]
        self.c0 = rng.randn(M, N).astype(np.float32)
        if c.get("nan_c0"):
            self.c0[:] = np.nan
        self.alpha, self.beta = c.get("alpha", 1.0), c.get("beta", 0.0)
        self.bias = torch.from_numpy(rng.randn(N).astype(np.float32)).cuda() if c.get("bias") else None
        self.relu = 1 if c.get("relu") else 0
        self.mask_np = self.mbuf = self.mask = None
        if c.get("mask"):
            moff = c.get("m_off", 0)
            self.mask_np = _mask_values(rng, M, N)
            self.mbuf = torch.zeros(moff + M * self.ldc + 4, dtype=torch.float32, device="cuda")
            self.mask = self.mbuf[moff:moff + M * self.ldc].view(M, self.ldc)
            self.mask[:, :N] = torch.from_numpy(self.mask_np).cuda()
        self.ws_bytes = lib.ctcb_gemm_workspace_bytes(M, N, K) if ws_bytes is None else ws_bytes
        self.ws = torch.full((self.ws_bytes + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")

    def plan(self):
        c = self.c
        return _plan(c["ta"], c["tb"], c["M"], c["N"], c["K"], self.a_ptr, self.lda, self.b_ptr, self.ldb)

    def run(self, null_ws=False):
        """Runs the contraction on C = C0 and returns C (NumPy)."""
        import _ctcb
        from _ctcb import lib, check, ptr
        c = self.c
        if self.C.numel():
            self.C.copy_(_torch().from_numpy(self.c0).cuda())
        check(lib.ctcb_gemm_f32(c["ta"], c["tb"], c["M"], c["N"], c["K"], self.alpha, self.a_ptr, self.lda, self.b_ptr,
                                self.ldb, self.beta, self.C.data_ptr(), self.ldc, ptr(self.bias),
                                self.relu, None if self.mask is None else self.mask.data_ptr(),
                                None if null_ws else ptr(self.ws), 0 if null_ws else self.ws_bytes,
                                _ctcb.current_stream()))
        _torch().cuda.synchronize()
        return self.C.cpu().numpy()

    def untouched(self):
        """Nothing outside C's M x N elements was written: C's padding and trailing rows, and the workspace guard."""
        torch = _torch()
        rest = self.cbuf.clone()
        coff = self.c.get("c_off", 0)
        M, N = self.c["M"], self.c["N"]
        rest[coff:coff + M * self.ldc].view(M, self.ldc)[:, :N] = SENTINEL
        ok_c = bool((rest == SENTINEL).all())
        ok_ws = bool((self.ws[self.ws_bytes:] == 0xA5).all())
        return ok_c, ok_ws

    def reference(self):
        """(C64, S) with the bias, ReLU and mask applied to C64."""
        M, N = self.c["M"], self.c["N"]
        if self.c["K"] > 0:
            P, S = _product(self.a_op, self.b_op)
        else:
            P, S = np.zeros((M, N)), np.zeros((M, N))
        want = self.alpha * P
        S = abs(self.alpha) * S
        if self.beta != 0.0:
            want = want + self.beta * self.c0.astype(np.float64)
            S = S + np.abs(self.beta * self.c0.astype(np.float64))
        if self.bias is not None:
            b = self.bias.cpu().numpy().astype(np.float64)
            want = want + b
            S = S + np.abs(b)
        if self.relu:
            want = np.maximum(want, 0.0)
        return want, S


def _compare(got, want, S, L, kernel, mask_np):
    """Element-wise error record; masked elements (not mask > 0) must be exactly 0."""
    c0, c1 = BOUNDS[kernel]
    keep = np.ones(got.shape, bool) if mask_np is None else (mask_np > 0)
    diff = np.abs(got.astype(np.float64) - want)
    lim = (c0 + c1 * L) * U * S
    ratio = np.where(S > 0, diff / np.maximum(U * S, 1e-300), np.where(diff > 0, np.inf, 0.0))
    rec = dict(L=L, ratio=float(ratio[keep].max()) if keep.any() else 0.0, bound=c0 + c1 * L,
               finite=bool(np.isfinite(got).all()))
    rec["within"] = bool((diff[keep] <= lim[keep]).all())
    if mask_np is not None:
        rec["masked_zero"] = bool((got[~keep] == 0).all())
        rec["denormal_kept"] = int(((mask_np == np.float32(1.4e-45)) & (got != 0)).sum())
    return rec


def _assert_rec(rec, what):
    assert rec["finite"], what
    assert rec.get("masked_zero", True), what
    assert rec["within"], (what, rec)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", list(CASES))
def test_gemm_plan(name, knobs, cuda):
    c = CASES[name]
    cuda.cuda.empty_cache()
    if c.get("simt"):
        knobs("CTCB_GEMM", "simt")
    if c.get("tc_copy"):
        knobs("CTCB_GEMM_TC_COPY", "1")
    call = Call(name, c)                          # workspace sized under the knobs just set
    plan = call.plan()
    _check_plan(plan, c["plan"], name)
    _check_ctas(plan, c["M"], c["N"])
    got = call.run()
    again = call.run()
    same = np.array_equal(got.view(np.uint32), again.view(np.uint32))
    ok_c, ok_ws = call.untouched()
    call.ws = None                                # room for the float64 reference of the largest cases
    want, S = call.reference()
    L = _chain(plan, c["K"])
    rec = _compare(got, want, S, L, plan["kernel"], call.mask_np)
    rec.update(plan=plan, same_bytes=same, c_untouched=ok_c, guard_untouched=ok_ws,
               peak_mb=round(cuda.cuda.max_memory_allocated() / 2 ** 20))
    print(json.dumps({"gemm_plan_" + name: rec}))
    assert same and ok_c and ok_ws, rec
    _assert_rec(rec, name)


# ---- workspaces short of the tensor-core need: the FFMA kernel, the same bits as CTCB_GEMM=simt with that workspace
WS_SHAPE = case(1, 0, 300, 200, 3000, None, beta=1.0, bias=True, mask=True)


@pytest.mark.parametrize("room", ["below_tc", "tiny", "null"])
def test_gemm_short_workspace_runs_ffma(room, knobs, cuda):
    from _ctcb import lib
    M, N, K = WS_SHAPE["M"], WS_SHAPE["N"], WS_SHAPE["K"]
    tc_need = lib.ctcb_gemm_workspace_bytes(M, N, K)
    ws_bytes = {"below_tc": tc_need - 256, "tiny": 256, "null": 0}[room]
    call = Call("ws", WS_SHAPE, ws_bytes=ws_bytes)
    _check_plan(call.plan(), dict(kernel=1), "ws")
    got = call.run(null_ws=room == "null")
    ok_c, ok_ws = call.untouched()
    knobs("CTCB_GEMM", "simt")
    simt_need = lib.ctcb_gemm_workspace_bytes(M, N, K)
    assert simt_need < tc_need - 256, (simt_need, tc_need)
    ref = Call("ws", WS_SHAPE, ws_bytes=ws_bytes)
    simt = ref.run(null_ws=room == "null")
    plan = ref.plan()
    # the FFMA plan at this workspace: split when the partials fit, else one chain over all of K
    if ws_bytes < simt_need:
        plan["splits"] = 1
    want, S = call.reference()
    rec = _compare(got, want, S, _chain(plan, K), 0, call.mask_np)
    rec.update(ws_bytes=ws_bytes, tc_need=tc_need, simt_need=simt_need, splits=plan["splits"],
               same_bytes=bool(np.array_equal(got.view(np.uint32), simt.view(np.uint32))),
               c_untouched=ok_c, guard_untouched=ok_ws)
    print(json.dumps({"gemm_ws_" + room: rec}))
    assert rec["same_bytes"] and ok_c and ok_ws, rec
    _assert_rec(rec, room)


# ---- the pair: one launch, or its fallbacks; each result is the single call's, byte for byte
PAIRS = {
    # name: (M = N = H, K, alpha, beta, A1 offset, workspace, expected plan of the pair)
    "one_launch": (512, 1568, 1.0, 1.0, 0, "pair", T(128, 6, MN, MN, problems=2)),
    "a1_off": (512, 1568, -0.5, 0.0, 1, "pair", T(128, 6, COPY, MN, problems=1)),
    "ws_between": (1024, 1000, 1.0, 1.0, 0, "single", T(128, 3, MN, MN, problems=2)),
    "ffma": (16, 1568, 1.0, 1.0, 0, "pair", F(11, 1)),
}


@pytest.mark.parametrize("name", list(PAIRS))
def test_gemm_pair_plans(name, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    H, K, alpha, beta, a1_off, room, expect = PAIRS[name]
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))
    ops = [torch.randn(K * H + 8, device="cuda", generator=gen) for _ in range(4)]
    A = [ops[0][:K * H].view(K, H), ops[1][a1_off:a1_off + K * H].view(K, H)]
    B = [ops[2][:K * H].view(K, H), ops[3][:K * H].view(K, H)]
    c0 = torch.randn(2, H, H, device="cuda", generator=gen)
    single_ws = lib.ctcb_gemm_workspace_bytes(H, H, K)
    pair_ws = lib.ctcb_gemm_pair_workspace_bytes(H, H, K)
    if room == "single":
        assert single_ws < pair_ws, (single_ws, pair_ws)
    ws_bytes = pair_ws if room == "pair" else single_ws
    ws = torch.full((ws_bytes + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    plan = _plan(1, 0, H, H, K, A[1].data_ptr(), H, B[1].data_ptr(), H, problems=2)
    _check_plan(plan, expect, name)
    _check_ctas(plan, H, H)
    st = _ctcb.current_stream()
    C = c0.clone()
    check(lib.ctcb_gemm_pair_f32(1, 0, H, H, K, alpha, A[0].data_ptr(), A[1].data_ptr(), H, B[0].data_ptr(),
                                 B[1].data_ptr(), H, beta, ptr(C[0]), ptr(C[1]), H, ptr(ws), ws_bytes, st))
    torch.cuda.synchronize()
    guard = bool((ws[ws_bytes:] == 0xA5).all())
    S1 = c0.clone()
    wss = torch.empty(single_ws, dtype=torch.uint8, device="cuda")
    for q in range(2):
        check(lib.ctcb_gemm_f32(1, 0, H, H, K, alpha, A[q].data_ptr(), H, B[q].data_ptr(), H, beta, ptr(S1[q]), H,
                                None, 0, None, ptr(wss), single_ws, st))
    torch.cuda.synchronize()
    same = bool(torch.equal(C.view(torch.int32), S1.view(torch.int32)))
    recs = []
    for q in range(2):
        P, S = _product(A[q].T, B[q])
        c0q = c0[q].cpu().numpy().astype(np.float64)
        want = alpha * P + beta * c0q
        S = abs(alpha) * S + abs(beta) * np.abs(c0q)
        qplan = _plan(1, 0, H, H, K, A[q].data_ptr(), H, B[q].data_ptr(), H)
        recs.append(_compare(C[q].cpu().numpy(), want, S, _chain(qplan, K), qplan["kernel"], None))
    print(json.dumps({"gemm_pair_" + name: dict(plan=plan, same_bytes=same, guard_untouched=guard, problems=recs)}))
    assert same and guard
    for q in range(2):
        _assert_rec(recs[q], (name, q))
