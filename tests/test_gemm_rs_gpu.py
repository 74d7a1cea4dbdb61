"""GPU unit test of what the tensor-core contraction's register path adds: the consumers read the A fragments of each
k-block from shared memory (128B-swizzled, a K-major box or four MN-major 32-row boxes) and split them into TF32 parts in
registers, and an MN-major A tile is read with its rows permuted (the epilogue puts them back).

Cases: M not a multiple of 64 (the second consumer's rows partly or wholly outside), K tails with K % 32 != 0 and
K % 8 != 0, A holding +-Inf, NaN, -0 and denormals, both problems of the pair with MN-major A, and tile widths 64 and 128
with K-major and MN-major A.  Every case checks its plan with ctcb_debug_gemm_plan and the element-wise bound of
test_gemm_plans_gpu.py, |C - C64| <= (c0 + c1 L) 2^-24 S, with its constants."""
import json
import zlib

import numpy as np
import pytest

from test_gemm_plans_gpu import KMAJOR, MN, T, BOUNDS, U, Call, case, _plan, _check_plan, _check_ctas, _chain, _compare, \
    _assert_rec

pytestmark = pytest.mark.gpu

CASES = {
    "m100_k203_bn128_kmajor": case(0, 1, 100, 96, 203, T(128, 1, KMAJOR, KMAJOR), bias=True),
    "m40_k203_bn64_mn": case(1, 0, 40, 64, 203, T(64, 1, MN, MN), beta=1.0),
    "m100_k300_bn64_kmajor_a": case(0, 0, 100, 64, 300, T(64, 1, KMAJOR, MN), relu=True, bias=True),
    "m300_k1000_bn64_mn_a": case(1, 1, 300, 50, 1000, T(64, 4, MN, KMAJOR), mask=True),
    "m200_k3003_bn128_mn": case(1, 0, 200, 200, 3003, T(128, 11, MN, MN), beta=1.0),
    "m260_k517_bn128_kmajor": case(0, 1, 260, 130, 517, T(128, 2, KMAJOR, KMAJOR), alpha=-0.5),
}


@pytest.mark.parametrize("name", list(CASES))
def test_gemm_rs_plan(name, cuda):
    c = CASES[name]
    call = Call(name, c)
    plan = call.plan()
    _check_plan(plan, c["plan"], name)
    _check_ctas(plan, c["M"], c["N"])
    got = call.run()
    ok_c, ok_ws = call.untouched()
    want, S = call.reference()
    rec = _compare(got, want, S, _chain(plan, c["K"]), 1, call.mask_np)
    rec.update(plan=plan, c_untouched=ok_c, guard_untouched=ok_ws)
    print(json.dumps({"gemm_rs_" + name: rec}))
    assert ok_c and ok_ws, rec
    _assert_rec(rec, name)


# A with special values.  x = hi + lo with hi the TF32 part: lo of +-Inf is Inf - Inf = NaN and lo of NaN is NaN, so a row of
# A holding one of them gives NaN in every column; -0 and denormals are ordinary values.
SPECIAL = {
    "kmajor": case(0, 1, 150, 100, 200, T(128, 1, KMAJOR, KMAJOR)),
    "mn": case(1, 0, 150, 100, 200, T(128, 1, MN, MN)),
}


@pytest.mark.parametrize("name", list(SPECIAL))
def test_gemm_rs_special_values(name, cuda):
    torch = cuda
    c = SPECIAL[name]
    call = Call("special_" + name, c)
    _check_plan(call.plan(), c["plan"], name)
    M, K = c["M"], c["K"]
    rng = np.random.RandomState(zlib.crc32(name.encode()) & 0x7fffffff)
    bad = {3: np.inf, 70: -np.inf, 131: np.nan}            # one row in each consumer's half of the tile, and the second tile
    a = call.a_op
    for m, v in bad.items():
        a[m, rng.randint(K)] = v
    fin = np.array([-0.0, 1.4e-45, -1.4e-45, 1.1754942e-38, -3e-40], dtype=np.float32)
    for m in (0, 64, 100, 149):                              # finite special values, spread over the row
        ks = rng.choice(K, size=(K // 2,), replace=False)
        a[m, torch.from_numpy(ks).cuda()] = torch.from_numpy(fin[rng.randint(len(fin), size=ks.size)]).cuda()
    a[5, :] = -0.0                                           # a row of -0 only
    got = call.run()
    rows = np.array(sorted(bad))
    assert np.isnan(got[rows]).all(), got[rows]
    keep = np.setdiff1d(np.arange(M), rows)
    want, S = call.reference()
    rec = _compare(got[keep], want[keep], S[keep], _chain(call.plan(), K), 1, None)
    print(json.dumps({"gemm_rs_special_" + name: rec}))
    _assert_rec(rec, name)
    assert (got[5] == 0).all()


# The recurrent weight-gradient pair: both problems MN-major in one launch, M = N = 200 (not a multiple of 64)
def test_gemm_rs_pair_mn(cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    H, K = 200, 1003
    gen = torch.Generator(device="cuda").manual_seed(5)
    A = [torch.randn(K, H, device="cuda", generator=gen) for _ in range(2)]
    B = [torch.randn(K, H, device="cuda", generator=gen) for _ in range(2)]
    plan = _plan(1, 0, H, H, K, A[1].data_ptr(), H, B[1].data_ptr(), H, problems=2)
    _check_plan(plan, T(128, 4, MN, MN, problems=2), "pair")
    _check_ctas(plan, H, H)
    ws = torch.empty(lib.ctcb_gemm_pair_workspace_bytes(H, H, K), dtype=torch.uint8, device="cuda")
    C = torch.zeros(2, H, H, device="cuda")
    check(lib.ctcb_gemm_pair_f32(1, 0, H, H, K, 1.0, A[0].data_ptr(), A[1].data_ptr(), H, B[0].data_ptr(),
                                 B[1].data_ptr(), H, 0.0, ptr(C[0]), ptr(C[1]), H, ptr(ws), ws.numel(),
                                 _ctcb.current_stream()))
    torch.cuda.synchronize()
    c0, c1 = BOUNDS[1]
    L = _chain(plan, K)
    for q in range(2):
        a, b = A[q].double().T, B[q].double()
        want, S = (a @ b).cpu().numpy(), (a.abs() @ b.abs()).cpu().numpy()
        diff = np.abs(C[q].cpu().numpy().astype(np.float64) - want)
        ratio = float((diff / (U * S)).max())
        print(json.dumps({"gemm_rs_pair_%d" % q: dict(L=L, ratio=ratio, bound=c0 + c1 * L)}))
        assert (diff <= (c0 + c1 * L) * U * S).all(), (q, ratio, c0 + c1 * L)
