"""GPU tests of the kernels the training step launches from csrc/brnn.cu itself, element-wise against float64 of their
own float32 inputs, and of every map's weight and bias gradients against the delta and input the step itself used.

a. Column sums (the bias gradients, ctcb_colsum_f32, the launches the step makes): |db - db64| <= C_COLSUM u D sum_r
   |delta_r|, u = 2^-24, with no floor.  D is the serial depth of the plan ctcb_debug_colsum_plan reports: wide path
   ceil(rpb / 4) + 2 + blocks (four row accumulators, their pairwise sum, the blocks' partials), narrow path 128 + 8 +
   blocks (a strided thread's rows, the 8 threads of a column, the partials); accumulate adds one level and u |prev|.
   C_COLSUM is 4x the largest ratio measured (below), a fifth of the worst case of a recursive sum.
b. Row softmax (ctcb_softmax_rows_f32, the launch of a forward-only call): |p - p64| <= C_SOFTMAX u p64 (max_k |x_k - m|
   + ceil(K / 32) + 8), plus C_SOFTMAX 2^-149 where p64 is below the normal range, against the float64 softmax of the
   float32 logits.  C_SOFTMAX = 2 a priori: x - m is rounded once (u |x - m| relative in exp), expf and the
   normaliser's lane and butterfly sums add ceil(K / 32) + 5 roundings, the reciprocal and the product two more.
c. Every affine map's gradients after one training call, from the step's own delta (ctcb_brnn_activation_offset what =
   7) and input (X_{j-1}, S for map L, the dropped activations under dropout): padded frames of the delta are +0.0,
   db_j meets bound (a) at the plan of its R(j) x rows(j) delta, dW_j meets the element-wise bound of
   test_gemm_plans_gpu.py at the plan ctcb_debug_gemm_plan reports.  A second micro-batch, without CTCB_PART_FIRST,
   must add its own sums onto the first's gradient under the same bounds with the first's values as C0.  The step's
   probabilities equal ctcb_softmax_rows_f32 of the logits it left behind, bit for bit.
d. The statistics tail, the L2 cost and gradient, ctcb_sumsq_f32, and For + Back at a bi-directional ReLU layer.
Each case prints its measured ratios to its bounds as one JSON line (pytest -s)."""
import ctypes
import json

import numpy as np
import pytest

import recipes
from net_check import bits
from test_gemm_plans_gpu import BOUNDS as GEMM_BOUNDS, FIELDS as GEMM_FIELDS, _chain as gemm_chain

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
# Measured on an H100 80GB HBM3 at 700 W: the largest |db - db64| / (u D sum|delta|) of the column-sum cases is 0.0410
# (wide_r5) and of the step's maps 0.0512 (map 4 of lstm_uni_peep_stack2); C_COLSUM is 4x the larger.  The worst case
# of a recursive sum, D u sum|x|, would allow 1 (2 with the remainder rows a wide block adds to its first accumulator).
C_COLSUM = 0.2
# A priori (module docstring); the largest ratio measured on an H100 80GB HBM3 at 700 W is 0.49 of it.
C_SOFTMAX = 2.0
NEG = 10.0                     # a wrong wiring must exceed the bound at least this many times
H100_SMS = 132
GUARD = 64                     # floats of NaN around every output
WS_GUARD = 4096                # bytes of 0xA5 behind every workspace
REACHED = dict(wide=False, narrow=False, lower=False, upper=False, interior=False, ncb=False, remainder=False)


def _ratio(err, bound):
    """max err / bound; NaN, or an error where the bound is 0, count as infinitely far."""
    err, bound = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(bound, np.float64))
    if not np.all(np.isfinite(err)) or np.any(err[bound <= 0.0] != 0.0):
        return float("inf")
    pos = bound > 0.0
    return float(np.max(err[pos] / bound[pos])) if pos.any() else 0.0


def _colsum_plan(R, n, ptr):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 4)()
    check(lib.ctcb_debug_colsum_plan(R, n, ptr, out))
    return dict(wide=out[0], ncb=out[1], rpb=out[2], blocks=out[3])


def _colsum_depth(plan):
    return (-(-plan["rpb"] // 4) + 2 if plan["wide"] else 128 + 8) + plan["blocks"]


def _colsum_bound(a, plan, prev=None):
    """C_COLSUM u D a, a = sum_r |delta_r| (+ one level and u |prev| when accumulating onto prev)."""
    if prev is None:
        return C_COLSUM * U * _colsum_depth(plan) * a
    prev = np.asarray(prev, np.float64)
    return C_COLSUM * U * (_colsum_depth(plan) + 1) * (a + np.abs(prev)) + U * np.abs(prev)


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ a. column sums
# name: (R, n, float offset of delta, expected plan on a 132-SM H100 {wide, ncb, rpb, blocks})
COLSUM_CASES = {
    "wide_lower_clamp": (6400, 512, 0, dict(wide=1, ncb=1, rpb=128, blocks=50)),
    "wide_interior_c3": (102400, 1024, 0, dict(wide=1, ncb=1, rpb=387, blocks=265)),
    "wide_upper_clamp": (300000, 64, 0, dict(wide=1, ncb=1, rpb=1024, blocks=293)),
    "wide_ncb4_lstm_gates": (20000, 4096, 0, dict(wide=1, ncb=4, rpb=303, blocks=67)),
    "wide_c4_hidden": (48000, 2048, 0, dict(wide=1, ncb=2, rpb=363, blocks=133)),
    "narrow_c4_output": (48000, 35, 0, dict(wide=0, ncb=2, rpb=1024, blocks=47)),
    "narrow_n1001": (5000, 1001, 0, dict(wide=0, ncb=32, rpb=1024, blocks=5)),
    "narrow_base_off": (7000, 512, 1, dict(wide=0, ncb=16, rpb=1024, blocks=7)),
    "wide_ragged_last": (6477, 256, 0, dict(wide=1, ncb=1, rpb=128, blocks=51)),
    "narrow_ragged_last": (3000, 35, 0, dict(wide=0, ncb=2, rpb=1024, blocks=3)),
    "wide_r1": (1, 64, 0, dict(wide=1, ncb=1, rpb=128, blocks=1)),
    "wide_r3": (3, 64, 0, dict(wide=1, ncb=1, rpb=128, blocks=1)),
    "wide_r5": (5, 64, 0, dict(wide=1, ncb=1, rpb=128, blocks=1)),
    "narrow_r1": (1, 33, 0, dict(wide=0, ncb=2, rpb=1024, blocks=1)),
    "narrow_r3": (3, 33, 0, dict(wide=0, ncb=2, rpb=1024, blocks=1)),
    "narrow_r5": (5, 33, 0, dict(wide=0, ncb=2, rpb=1024, blocks=1)),
}


def _delta_rows(seed, R, n):
    """randn rows of mixed scale, every seventh row 0 (a padded frame), a few rows 1000x."""
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((R, n), dtype=np.float32)
    d *= rng.uniform(0.01, 2.0, size=(R, 1)).astype(np.float32)
    d[3::7] = 0.0
    d[5::97] *= np.float32(1000.0)
    return d


def _sums64(d, chunk=4096):
    """(sum, sum of |.|) over the rows of float32 d in float64, a chunk of rows at a time."""
    s = np.zeros(d.shape[1])
    a = np.zeros(d.shape[1])
    for r0 in range(0, d.shape[0], chunk):
        x = d[r0:r0 + chunk].astype(np.float64)
        s += x.sum(axis=0)
        a += np.abs(x).sum(axis=0)
    return s, a


@pytest.mark.parametrize("name", list(COLSUM_CASES))
def test_colsum_matches_float64(name, cuda):
    torch = cuda
    import _ctcb
    from _ctcb import lib, check
    R, n, off, expect = COLSUM_CASES[name]
    rng = np.random.RandomState(R * 7 + n)
    d = _delta_rows(R * 7 + n, R, n)
    buf = torch.zeros(R * n + off + 4, dtype=torch.float32, device="cuda")
    buf[off:off + R * n] = torch.from_numpy(d.reshape(-1)).cuda()
    dptr = buf.data_ptr() + 4 * off
    plan = _colsum_plan(R, n, dptr)
    if plan != expect:
        msg = "%s: planned %s, this case targets %s" % (name, plan, expect)
        if _sms(torch) != H100_SMS:
            pytest.skip("plan not reachable on this device: " + msg)
        pytest.fail(msg)
    sms = _sms(torch)
    if plan["wide"]:                   # the planner's rule, restated
        rpb = min(max(R // max(1, 2 * sms // plan["ncb"]), 128), 1024)
        assert plan["rpb"] == rpb and plan["blocks"] == -(-R // rpb), plan
    ws_bytes = int(lib.ctcb_colsum_workspace_bytes(R, n))
    assert ws_bytes == -(-R // 128) * n * 4
    ws = torch.full((ws_bytes + WS_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    prev = (rng.randn(n) * 50).astype(np.float32)
    st = _ctcb.current_stream()
    outs = {}
    for acc in (0, 1, 0):
        o = torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
        if acc:
            o[GUARD:GUARD + n] = torch.from_numpy(prev).cuda()
        check(lib.ctcb_colsum_f32(dptr, R, n, o.data_ptr() + 4 * GUARD, acc, ws.data_ptr(), ws_bytes, st))
        torch.cuda.synchronize()
        h = o.cpu().numpy()
        assert np.isnan(h[:GUARD]).all() and np.isnan(h[GUARD + n:]).all(), "wrote outside out"
        if acc in outs:
            assert np.array_equal(h.view(np.uint32), outs[acc].view(np.uint32)), "a rerun gave other bytes"
        outs[acc] = h
    assert bool((ws[ws_bytes:] == 0xA5).all()), "wrote past the workspace"
    del buf
    want, a = _sums64(d)
    r = _ratio(np.abs(outs[0][GUARD:GUARD + n] - want), _colsum_bound(a, plan))
    r_acc = _ratio(np.abs(outs[1][GUARD:GUARD + n] - (want + prev)), _colsum_bound(a, plan, prev))
    print(json.dumps({"colsum_" + name: dict(plan=plan, depth=_colsum_depth(plan), ratio=r, ratio_acc=r_acc,
                                             c=C_COLSUM)}))
    assert r <= 1.0 and r_acc <= 1.0, (r, r_acc)
    REACHED["wide" if plan["wide"] else "narrow"] = True
    if plan["wide"]:
        REACHED["lower"] |= plan["rpb"] == 128 and R >= 128
        REACHED["upper"] |= plan["rpb"] == 1024
        REACHED["interior"] |= 128 < plan["rpb"] < 1024
        REACHED["ncb"] |= plan["ncb"] > 1
        REACHED["remainder"] |= plan["rpb"] % 4 != 0


# ------------------------------------------------------------------------------------------------ b. softmax
def _softmax_rows(rng, R, K):
    """Logits of every kind: randn x 3, equal logits, a repeated maximum, near +1e4 and -1e4, spreads of about 100
    (probabilities down to the subnormals and 0)."""
    x = (3.0 * rng.randn(R, K)).astype(np.float32)
    kinds = np.arange(R) % 7
    x[kinds == 1] = np.float32(0.37)
    rep = np.where(kinds == 2)[0]
    for r in rep:
        x[r, :min(K, 3)] = x[r].max() + 1.0
    x[kinds == 3] = (1e4 + rng.randn(int((kinds == 3).sum()), K)).astype(np.float32)
    x[kinds == 4] = (-1e4 + rng.randn(int((kinds == 4).sum()), K)).astype(np.float32)
    x[kinds == 5] = rng.uniform(-100.0, 0.0, size=(int((kinds == 5).sum()), K)).astype(np.float32)
    x[kinds == 6] = rng.uniform(-120.0, 5.0, size=(int((kinds == 6).sum()), K)).astype(np.float32)
    return x


def _softmax_check(x, p):
    """(ratio to the bound, p64) of float32 probabilities p against the float64 softmax of float32 logits x."""
    x64 = x.astype(np.float64)
    m = x64.max(axis=1, keepdims=True)
    e = np.exp(x64 - m)
    p64 = e / e.sum(axis=1, keepdims=True)
    K = x.shape[1]
    bound = C_SOFTMAX * U * p64 * (np.abs(x64 - m).max(axis=1, keepdims=True) + -(-K // 32) + 8)
    bound = bound + np.where(p64 < 2.0 ** -126, C_SOFTMAX * 2.0 ** -149, 0.0)
    return _ratio(np.abs(p.astype(np.float64) - p64), bound), p64


@pytest.mark.parametrize("K", [1, 31, 32, 33, 62, 64, 65, 1000])
@pytest.mark.parametrize("R", [1, 1003])
def test_softmax_rows_match_float64(R, K, cuda):
    torch = cuda
    import _ctcb
    from _ctcb import lib, check
    rng = np.random.RandomState(R * 1000 + K)
    x = _softmax_rows(rng, R, K)
    dx = torch.from_numpy(x).cuda()
    p = torch.full((R * K + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    st = _ctcb.current_stream()
    check(lib.ctcb_softmax_rows_f32(dx.data_ptr(), p.data_ptr() + 4 * GUARD, R, K, st))
    h = p.cpu().numpy()
    assert np.isnan(h[:GUARD]).all() and np.isnan(h[GUARD + R * K:]).all(), "wrote outside p"
    got = h[GUARD:GUARD + R * K].reshape(R, K)
    r, p64 = _softmax_check(x, got)
    p2 = torch.empty(R * K, dtype=torch.float32, device="cuda")
    check(lib.ctcb_softmax_rows_f32(dx.data_ptr(), p2.data_ptr(), R, K, st))
    same = np.array_equal(bits(p2), got.reshape(-1).view(np.uint32))
    sub = int(((p64 > 0) & (p64 < 2.0 ** -126)).sum())
    print(json.dumps({"softmax_R%d_K%d" % (R, K): dict(ratio=r, c=C_SOFTMAX, subnormal_p64=sub, same_bytes=same)}))
    assert r <= 1.0, r
    assert same
    if K == 1:
        assert (got == 1.0).all()
    eq = np.where(np.arange(R) % 7 == 1)[0]
    if len(eq):                            # equal logits: every probability of the row is the same float
        assert (got[eq] == got[eq][:, :1]).all()


# ------------------------------------------------------------------------------------------------ c. every map's gradients
D_IN = 23
NETS = {
    # name: NNet keyword arguments, layer size, hidden layers, output width
    "bi_relu_k35": dict(H=64, N=3, K=35, kw=dict(temporalLayer=2)),
    "uni_relu_stack3": dict(H=48, N=4, K=29, kw=dict(temporalLayer=1, numTemporal=3, unidirectional=True)),
    "bi_relu_stack2": dict(H=64, N=3, K=30, kw=dict(temporalLayer=1, numTemporal=2)),
    "dnn_h70_ln": dict(H=70, N=3, K=31, kw=dict(layerNorm=True)),
    "lstm_bi": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm")),
    "lstm_uni_peep_stack2": dict(H=33, N=3, K=28, kw=dict(temporalLayer=1, numTemporal=2, cell="lstm",
                                                         unidirectional=True, peephole=True)),
    "bi_ln_dropout": dict(H=64, N=3, K=33, kw=dict(temporalLayer=2, layerNorm=True, dropout=0.1)),
    "uni_sub2_L2": dict(H=64, N=3, K=30, kw=dict(temporalLayer=2, unidirectional=True, subsample=2,
                                                  subsampleLayer=2)),
    "bi_sub3_L3_dropout": dict(H=44, N=3, K=27, kw=dict(temporalLayer=2, subsample=3, subsampleLayer=3,
                                                         dropout=0.1)),
    # the recurrent and peephole gradients of both directions through the zoneout sweep's BPTT
    "lstm_bi_peep_zoneout": dict(H=32, N=3, K=28, kw=dict(temporalLayer=2, cell="lstm", peephole=True,
                                                          zoneoutCell=0.2, zoneoutHidden=0.15)),
}
MAXT, MAXB = 40, 7


def _net(c):
    import nnets.brnnet as brnnet
    np.random.seed(17)
    nn = brnnet.NNet(D_IN, c["K"], c["H"], c["N"], MAXT, maxUtts=MAXB, maxLabels=6, **c["kw"])
    nn.initParams()
    rng = np.random.RandomState(2)        # biases off 0, so a padded frame's activations are not 0 on their own
    for w, b in nn.stack[:c["N"] + 1]:
        b.copy_(nn._torch.from_numpy((0.1 * rng.randn(*b.shape)).astype(np.float32)))
    return nn


def _hook(nn, what, layer):
    """(byte offset, width) of the activation hook, or None where it refuses."""
    from _ctcb import lib
    off, width = ctypes.c_size_t(), ctypes.c_int32()
    if lib.ctcb_brnn_activation_offset(ctypes.byref(nn._cfg), what, layer, ctypes.byref(off), ctypes.byref(width)):
        return None
    return off.value, width.value


def _ws_array(nn, off, T, B, n):
    torch = nn._torch
    return nn._ws[off:off + 4 * T * B * n].view(torch.float32).view(T, B, n)


def _map_input(nn, j, batch):
    """(device [T][B][cols] float32 of the input X_{j-1} that map j's weight gradient read, pointer for the plan)."""
    T = nn.frames(batch.Tmax) if nn.subsample > 1 and j >= nn.subsampleLayer else batch.Tmax
    B = batch.B
    if nn.subsample > 1 and j == nn.subsampleLayer:
        off, w = _hook(nn, 6, 0)
        x = _ws_array(nn, off, T, B, w)
        return x, x.data_ptr()
    if j == 1:
        x = batch.d_feats[:T * B * nn.inputDim].view(T, B, nn.inputDim)
        return x, x.data_ptr()
    i = j - 1
    tl, k = nn.temporalLayer, nn.numTemporal
    temporal = k and tl <= i < tl + k
    if temporal and nn.unidirectional:
        off, w = _hook(nn, 1, i)
        x = _ws_array(nn, off, T, B, w)
        return x, x.data_ptr()
    if temporal and nn.cell == "lstm":      # For + Back in float32, as the step's add2 (Out is not exposed)
        off1, w = _hook(nn, 1, i)
        off2, _ = _hook(nn, 2, i)
        hf = _ws_array(nn, off1, T, B, w)
        return hf + _ws_array(nn, off2, T, B, w), hf.data_ptr()
    off, w = _hook(nn, 0, i)
    x = _ws_array(nn, off, T, B, w)
    return x, x.data_ptr()


def _gemm_plan(M, N, K, a_ptr, lda, b_ptr, ldb):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan(1, 0, M, N, K, a_ptr, lda, b_ptr, ldb, 1, out))
    return dict(zip(GEMM_FIELDS, list(out)))


def _check_maps(nn, batch, lens, prev=None, neg=None):
    """Every map's padded delta frames, db and dW against the call's own delta and input, and the recurrent (and
    peephole) gradients of every LSTM layer and of the lowest two of a uni-directional ReLU stack (rec_grads).  prev:
    the flat gradient (float32, NumPy) the call added onto, or None for a CTCB_PART_FIRST call.  neg collects the
    negative controls.  Returns {map: ratios}."""
    B, N = batch.B, nn.numLayers
    grads = nn.grads.cpu().numpy()
    out = {}
    for j in range(1, N + 2):
        reduced = nn.subsample > 1 and j >= nn.subsampleLayer
        T = nn.frames(batch.Tmax) if reduced else batch.Tmax
        Tu = [nn.frames(t) if reduced else t for t in lens]
        h = _hook(nn, 7, j)
        tl, k = nn.temporalLayer, nn.numTemporal
        if h is None:        # only where a lower layer of a uni-directional ReLU stack writes the same pair
            assert nn.unidirectional and nn.cell == "relu" and k and j - tl >= 2, j
            out[j] = "overwritten"
            continue
        off, rows = h
        assert rows == nn._map_rows(j)
        dd = _ws_array(nn, off, T, B, rows)
        d = dd.cpu().numpy()
        for u in range(B):
            assert not d[Tu[u]:, u].view(np.uint32).any(), "map %d: a padded frame of the delta is not +0.0" % j
        R = T * B
        d64 = d.reshape(R, rows).astype(np.float64)
        x, xptr = _map_input(nn, j, batch)
        cols = x.shape[2]
        x64 = x.cpu().numpy().reshape(R, cols).astype(np.float64)
        wv, bv = nn.grad[j - 1]
        w_off = (wv.data_ptr() - nn.grads.data_ptr()) // 4
        b_off = (bv.data_ptr() - nn.grads.data_ptr()) // 4
        dw = grads[w_off:w_off + rows * cols].reshape(rows, cols).astype(np.float64)
        db = grads[b_off:b_off + rows].astype(np.float64)
        cplan = _colsum_plan(R, rows, dd.data_ptr())
        gplan = _gemm_plan(rows, cols, R, dd.data_ptr(), rows, xptr, cols)
        L = gemm_chain(gplan, R)
        c0, c1 = GEMM_BOUNDS[gplan["kernel"]]
        P, S = d64.T @ x64, np.abs(d64).T @ np.abs(x64)
        want_b = d64.sum(axis=0)
        if prev is None:
            bound_b = _colsum_bound(np.abs(d64).sum(axis=0), cplan)
        else:
            pw = prev[w_off:w_off + rows * cols].reshape(rows, cols).astype(np.float64)
            pb = prev[b_off:b_off + rows].astype(np.float64)
            P, S = P + pw, S + np.abs(pw)
            want_b = want_b + pb
            bound_b = _colsum_bound(np.abs(d64).sum(axis=0), cplan, pb)
        r_w = _ratio(np.abs(dw - P), (c0 + c1 * L) * U * S)
        r_b = _ratio(np.abs(db - want_b), bound_b)
        out[j] = dict(R=R, rows=rows, cols=cols, colsum=cplan, gemm_kernel=gplan["kernel"], L=L, dW=r_w, db=r_b)
        assert r_w <= 1.0 and r_b <= 1.0, (j, out[j])
    for j in range(nn.numTemporal):      # the recurrent gradients, where the delta they read survives the call
        if nn.cell == "relu" and not (nn.unidirectional and j < 2):
            continue
        r = _rec_from_hooks(nn, batch, lens, j, grads, prev, neg)
        out["rec%d" % (nn.temporalLayer + j)] = r
        assert max(v for k, v in r.items() if not k.startswith("kernel")) <= 1.0, (j, r)
    return out


def _rec_from_hooks(nn, batch, lens, j, grads, prev, neg):
    """rec_grads of temporal layer tl + j from what the call left: dz (LSTM) or dFor (uni-directional ReLU, j < 2),
    For / Back and Cf / Cb."""
    i = nn.temporalLayer + j
    reduced = nn.subsample > 1 and i >= nn.subsampleLayer
    T = nn.frames(batch.Tmax) if reduced else batch.Tmax
    Tu = [nn.frames(t) if reduced else t for t in lens]
    B, H = batch.B, nn.layerSize
    ndir = 1 if nn.unidirectional else 2
    dd = _ws_array(nn, _hook(nn, 7, i)[0], T, B, nn._map_rows(i))
    d = dd.cpu().numpy()
    hd = [_ws_array(nn, _hook(nn, 1 + q, i)[0], T, B, H) for q in range(ndir)]
    hs = [x.cpu().numpy() for x in hd]
    if nn.cell == "lstm":
        M = 4 * H
        dzs = [d[:, :, q * M:(q + 1) * M] for q in range(ndir)]
        cs = [_ws_array(nn, _hook(nn, 4 + q, i)[0], T, B, H).cpu().numpy() for q in range(ndir)]
        ldz = ndir * M
        ptrs = (dd.data_ptr() + 4 * B * ldz, dd.data_ptr() + 4 * M, hd[0].data_ptr(),
                hd[-1].data_ptr() + 4 * B * H, ldz)
    else:
        dzs, cs = [d], None
        ptrs = (dd.data_ptr() + 4 * B * H, None, hd[0].data_ptr(), None, H)
    return rec_grads(nn, j, T, Tu, dzs, hs, cs, ptrs, grads, prev, neg)


def _grad_view(nn, grads, idx, part=0):
    """float64 copy of tensor stack[idx][part] of the flat float32 gradient `grads` (NumPy)."""
    v = nn.grad[idx][part]
    o = (v.data_ptr() - nn.grads.data_ptr()) // 4
    return grads[o:o + v.numel()].reshape(tuple(v.shape))


def _pairs(T, Tu, d):
    """[T][B] weights of the frames t whose dz direction d pairs with h of frame t - 1 (d = 0) or t + 1 (d = 1) in
    its own utterance: 0 where that frame lies outside [0, T_u)."""
    t = np.arange(T)[:, None]
    Tu = np.asarray(Tu)[None, :]
    return ((t < Tu) & (t >= 1) if d == 0 else (t + 1 < Tu)).astype(np.float64)


def _shift(x, d):
    """x [T][B][n] moved one frame: y[t] = x[t - 1] (d = 0) or x[t + 1] (d = 1), 0 beyond the ends."""
    y = np.zeros(x.shape)
    if d == 0:
        y[1:] = x[:-1]
    else:
        y[:-1] = x[1:]
    return y


def peep_idx(nn, j, d):
    """Index into nn.stack of [P, dummy] of direction d of temporal layer tl + j."""
    ndir = 1 if nn.unidirectional else 2
    return len(nn.stack) - (1 if nn.selfCondition else 0) - nn.peepholeEntries() + j * ndir + d


def rec_grads(nn, j, T, Tu, dzs, hs, cs, ptrs, grads, prev=None, neg=None):
    """Ratios of the recurrent weight gradients of temporal layer tl + j (dU, or Wtf / Wtb) and of its peephole
    gradients to float64 of the float32 deltas dzs and states hs, cs (per direction [T][B][.], direction 1 reversed in
    time), each direction paired with its own shift within each utterance's length T_u.  The contraction: the bound of
    test_gemm_plans_gpu.py at each problem's plan, as test_gemm_pair_plans takes it (ptrs: the step's A0, A1, B0, B1
    and the pitch of A); dP: the bound of test_peephole_grad_matches_float64.  prev: the flat gradient the call added
    onto (None for CTCB_PART_FIRST).  One frame: the recurrent gradients are exactly +0.0 in a first part and keep
    their bytes in an accumulating one.  neg collects the negative controls: direction 1 unshifted, dp_o with c_prev,
    beta = 0 where the call accumulates."""
    ndir = len(dzs)
    H = hs[0].shape[2]
    B = hs[0].shape[1]
    M = dzs[0].shape[2]
    base = nn.numLayers + 1 + j * ndir
    out = {}
    neg = {} if neg is None else neg
    lda = ptrs[4]
    for d in range(ndir):
        w = _pairs(T, Tu, d)[:, :, None]
        A = (dzs[d].astype(np.float64) * w).reshape(T * B, M)
        Bm = _shift(hs[d].astype(np.float64), d).reshape(T * B, H)
        P, S = A.T @ Bm, np.abs(A).T @ np.abs(Bm)
        got = _grad_view(nn, grads, base + d).astype(np.float64)
        pw = None if prev is None else _grad_view(nn, prev, base + d).astype(np.float64)
        if T == 1:                       # no recurrence: a memset in a first part, untouched in an accumulating one
            want = np.zeros_like(got) if pw is None else pw
            out["dU%d" % d] = 0.0 if np.array_equal(got.astype(np.float32).view(np.uint32),
                                                     want.astype(np.float32).view(np.uint32)) else float("inf")
        else:
            a_ptr, b_ptr = (ptrs[0], ptrs[2]) if d == 0 else (ptrs[1], ptrs[3])
            plan = _gemm_plan(M, H, (T - 1) * B, a_ptr, lda, b_ptr, H)
            c0, c1 = GEMM_BOUNDS[plan["kernel"]]
            k = (c0 + c1 * gemm_chain(plan, (T - 1) * B)) * U
            if pw is not None and pw.any():      # (after a part of one-frame utterances dU is 0)
                neg.setdefault("beta_0_accumulating", []).append(_ratio(np.abs(got - P), k * (S + np.abs(pw))))
                P, S = P + pw, S + np.abs(pw)
            out["dU%d" % d] = _ratio(np.abs(got - P), k * S)
            out["kernel%d" % d] = plan["kernel"]
            if d == 1:
                wrong = dzs[d].astype(np.float64).reshape(T * B, M).T @ hs[d].astype(np.float64).reshape(T * B, H)
                neg.setdefault("direction_1_unshifted", []).append(_ratio(np.abs(got - wrong - (0 if pw is None else pw)),
                                                                          k * S))
        if not nn.peephole:
            continue
        dz = dzs[d].astype(np.float64)
        live = (np.arange(T)[:, None] < np.asarray(Tu)[None, :])[:, :, None]
        c = cs[d].astype(np.float64) * live
        cp = _shift(c, d) * _pairs(T, Tu, d)[:, :, None]
        terms = [dz[:, :, :H] * cp, dz[:, :, H:2 * H] * cp, dz[:, :, 3 * H:] * c]
        want = np.stack([x.sum(axis=(0, 1)) for x in terms])
        S = np.stack([np.abs(x).sum(axis=(0, 1)) for x in terms])
        K = 128 + 8 + -(-(T * B) // 1024) + 1
        bound = K * U * S
        ip = peep_idx(nn, j, d)
        got = _grad_view(nn, grads, ip).astype(np.float64)
        if prev is not None:
            pp = _grad_view(nn, prev, ip).astype(np.float64)
            neg.setdefault("beta_0_accumulating", []).append(_ratio(np.abs(got - want), bound + U * np.abs(want + pp)))
            want = want + pp
            bound = bound + U * np.abs(want)
        out["dP%d" % d] = _ratio(np.abs(got - want), bound)
        wrong = want.copy()
        wrong[2] += (dz[:, :, 3 * H:] * (cp - c)).sum(axis=(0, 1))
        neg.setdefault("dp_o_with_c_prev", []).append(_ratio(np.abs(got - wrong), bound))
        if d == 1:
            wrong = want.copy()
            wrong[:2] += np.stack([(dz[:, :, q * H:(q + 1) * H] * (c - cp)).sum(axis=(0, 1)) for q in range(2)])
            neg.setdefault("direction_1_unshifted", []).append(_ratio(np.abs(got - wrong), bound))
    return out


def _batches(c, seed):
    rng = np.random.RandomState(seed)
    lens = [int(t) for t in rng.randint(3, MAXT - 4, size=MAXB)]
    lens[1] = MAXT - 3
    lens[-1] = 1 if seed % 2 else 2                  # a one- or two-frame utterance: all padding after it
    nlabs = [int(x) for x in rng.randint(1, 3, size=MAXB)]
    nlabs[-1] = 1
    return lens, recipes.synth_batch(D_IN, c["K"], lens, nlabs, seed=seed)


@pytest.mark.parametrize("name", list(NETS))
def test_every_map_gradient_from_the_step_delta(name, cuda):
    torch = cuda
    from _ctcb import lib, check
    import _ctcb
    c = NETS[name]
    nn = _net(c)
    nn.grads.fill_(float("nan"))                      # CTCB_PART_FIRST must overwrite every tensor
    rep, neg = {}, {}
    prev = None
    u0 = 0
    for part, seed in enumerate((41, 42)):
        lens, (datas, labelss) = _batches(c, seed)
        batch = nn.swap_batches().pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, want_probs=True, first=part == 0, last=part == 1, u0=u0)
        u0 += batch.B
        torch.cuda.synchronize()
        rep[part] = _check_maps(nn, batch, lens, prev, neg)
        # the probabilities the call wrote are the softmax of the logits it left behind, bit for bit
        T = nn.frames(batch.Tmax)
        off, K = _hook(nn, 0, nn.numLayers + 1)
        logits = _ws_array(nn, off, T, batch.B, K)
        p = torch.empty(T * batch.B * K, dtype=torch.float32, device="cuda")
        check(lib.ctcb_softmax_rows_f32(logits.data_ptr(), p.data_ptr(), T * batch.B, K, _ctcb.current_stream()))
        assert np.array_equal(bits(p), bits(nn._probs_view(batch.B, T)).reshape(-1)), "probs_out != softmax(logits)"
        prev = nn.grads.cpu().numpy().copy()
    # the dummy biases of the recurrent matrices and of the peephole vectors receive exactly 0
    nmaps = nn.numLayers + 1
    ndir = 1 if nn.unidirectional else 2
    dummies = [nn.grad[p][1] for p in range(nmaps, nmaps + nn.numTemporal * ndir)]
    dummies += [nn.grad[-1 - q][1] for q in range(nn.peepholeEntries())]
    assert all(bool((d == 0).all()) for d in dummies), "a dummy bias has a gradient"
    negs = {k: min(v) for k, v in neg.items()}
    print(json.dumps({"step_maps_" + name: {"first": rep[0], "accumulate": rep[1], "negative_controls": negs}}))
    assert all(v >= NEG for v in negs.values()), negs


def _one_frame_batch(c, seed):
    """MAXB utterances of one frame and one label each."""
    lens = [1] * MAXB
    return lens, recipes.synth_batch(D_IN, c["K"], lens, [1] * MAXB, seed=seed)


@pytest.mark.parametrize("name", [n for n, c in NETS.items() if c["kw"].get("temporalLayer")])
def test_one_frame_micro_batches(name, cuda):
    """A micro-batch whose utterances are all one frame long (Tmax = 1: no recurrence): as a first part every recurrent
    gradient is exactly +0.0; after a part of full-length utterances, as an accumulating part, the recurrent gradients
    keep their bytes and dP adds the dz_o c term alone; every map's gradients meet part (c)'s bounds throughout."""
    torch = cuda
    c = NETS[name]
    nn = _net(c)
    nn.grads.fill_(float("nan"))
    rep, neg = {}, {}
    prev = None
    u0 = 0
    for part, (kind, seed) in enumerate((("ones", 44), ("full", 41), ("ones", 45))):
        lens, (datas, labelss) = (_one_frame_batch if kind == "ones" else _batches)(c, seed)
        batch = nn.swap_batches().pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, first=part == 0, last=part == 2, u0=u0)
        u0 += batch.B
        torch.cuda.synchronize()
        assert (batch.Tmax == 1) == (kind == "ones")
        rep[part] = _check_maps(nn, batch, lens, prev, neg)
        prev = nn.grads.cpu().numpy().copy()
    ndir = 1 if nn.unidirectional else 2
    rec = [_grad_view(nn, prev, nn.numLayers + 1 + q) for q in range(nn.numTemporal * ndir)]
    negs = {k: min(v) for k, v in neg.items()}
    print(json.dumps({"step_one_frame_" + name: dict(parts=rep, negative_controls=negs)}))
    assert all(v >= NEG for v in negs.values()), negs
    assert all(np.isfinite(x).all() for x in rec)


# ------------------------------------------------------------------------------------------------ d. the tail
def _tail_net(maxB, reg=0.0, **kw):
    import nnets.brnnet as brnnet
    np.random.seed(5)
    nn = brnnet.NNet(13, 11, 32, 2, 24, maxUtts=maxB, maxLabels=12, reg=reg, **kw)
    nn.initParams()
    return nn


def _tail_batch(B, seed):
    """B utterances of 2..24 frames with at most T / 2 labels; every fifth is 4 frames of the labels 3 3 3, which need 5
    (a blank between repeats), so the CTC finds no alignment and skips it."""
    rng = np.random.RandomState(seed)
    lens = [int(t) for t in rng.randint(2, 25, size=B)]
    nlabs = [int(max(1, min(t // 2, x))) for t, x in zip(lens, rng.randint(1, 6, size=B))]
    for u in range(0, B, 5):
        lens[u], nlabs[u] = 4, 3
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=seed)
    for u in range(0, B, 5):
        labelss[u] = np.array([3, 3, 3], np.int32)
    return datas, labelss


@pytest.mark.parametrize("B", [1, 33, 100])
def test_statistics_tail(B, cuda):
    torch = cuda
    nn = _tail_net(100)
    want = np.zeros(4)
    tot_abs, depth = 0.0, 0
    for part, seed in enumerate((7, 8)):
        datas, labelss = _tail_batch(B, seed + B)
        batch = nn.swap_batches().pack(datas, labelss).upload()
        cost, skip = nn.costAndGradDevice(batch, first=part == 0, last=part == 1)
        torch.cuda.synchronize()
        cost = cost.cpu().numpy().astype(np.float64)
        skip = skip.cpu().numpy() != 0
        assert skip[0] and skip.sum() == len(range(0, B, 5)), skip
        ok = ~skip
        assert np.isfinite(cost[ok]).all()
        want += [ok.sum(), cost[ok].sum(), skip.sum(), 0.0]
        tot_abs += np.abs(cost[ok]).sum()
        depth += B
        stats = nn.stats.cpu().numpy().astype(np.float64)
        assert stats[0] == want[0] and stats[2] == want[2] and stats[3] == 0.0, (stats, want)
        r = _ratio(abs(stats[1] - want[1]), (depth + part) * U * tot_abs)
        print(json.dumps({"stats_B%d_part%d" % (B, part): dict(stats=stats.tolist(), want=want.tolist(), ratio=r)}))
        assert r <= 1.0, (stats, want)


def test_regcost_l2_gradient_and_sumsq(cuda):
    torch = cuda
    import _ctcb
    from _ctcb import lib, check, ptr
    reg = float(np.float32(0.03))
    nn = _tail_net(8, reg=reg, temporalLayer=1, layerNorm=True)
    rng = np.random.RandomState(3)
    nn.params.copy_(torch.from_numpy(rng.randn(nn.nparams).astype(np.float32)))
    datas, labelss = _tail_batch(8, 3)
    nn.costAndGradBatch(datas, labelss)
    # regcost: 0.5 reg sum over the weight matrices (the maps' W and the recurrent matrices) of |W|^2
    widx = list(range(0, 2 * (nn.numLayers + 1), 2)) + [2 * (nn.numLayers + 1)] + [2 * (nn.numLayers + 1) + 2]
    ws = [nn.stack[i // 2][0].cpu().numpy().astype(np.float64) for i in widx]
    want = 0.5 * reg * sum((w ** 2).sum() for w in ws)
    got = float(nn._regcost.item())
    r_reg = abs(got - want) / (4 * (len(ws) + 1) * U * want)
    # the L2 gradient: g + reg W on those matrices, every other tensor unchanged
    g0 = torch.from_numpy(rng.randn(nn.nparams).astype(np.float32)).cuda()
    g = g0.clone()
    check(lib.ctcb_brnn_apply_l2_f32(nn._h, ptr(nn.params), ptr(g), _ctcb.current_stream()))
    gv, pv, g0v = nn._views(g), nn.stack, nn._views(g0)
    r_l2 = 0.0
    for t in range(2 * len(nn.stack)):
        a, b = gv[t // 2][t % 2].cpu().numpy(), g0v[t // 2][t % 2].cpu().numpy()
        if t in widx:
            w = pv[t // 2][t % 2].cpu().numpy().astype(np.float64)
            e = np.abs(a - (b.astype(np.float64) + reg * w))
            r_l2 = max(r_l2, _ratio(e, 2 * U * (np.abs(b) + reg * np.abs(w))))
        else:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), t
    # sumsq of n = 10^6 + 3 floats against float64
    v = rng.randn(1000003).astype(np.float32) * rng.uniform(0.1, 10.0, size=1000003).astype(np.float32)
    dv = torch.from_numpy(v).cuda()
    out = torch.zeros(1, dtype=torch.float32, device="cuda")
    scratch = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    check(lib.ctcb_sumsq_f32(ptr(dv), v.size, ptr(out), ptr(scratch), _ctcb.current_stream()))
    s64 = float((v.astype(np.float64) ** 2).sum())
    r_ss = abs(float(out.item()) - s64) / (4 * U * s64)
    print(json.dumps({"tail_reg_l2_sumsq": dict(regcost=r_reg, l2=r_l2, sumsq=r_ss)}))
    assert r_reg <= 1.0 and r_l2 <= 1.0 and r_ss <= 1.0, (r_reg, r_l2, r_ss)


def test_bidirectional_relu_output_is_for_plus_back(cuda):
    torch = cuda
    nn = _net(NETS["bi_relu_stack2"])
    lens, (datas, labelss) = _batches(NETS["bi_relu_stack2"], 43)
    nn.costAndGradBatch(datas, labelss)
    torch.cuda.synchronize()
    T, B = max(lens), len(lens)
    for i in (nn.temporalLayer, nn.temporalLayer + 1):
        x = _ws_array(nn, *_hook(nn, 0, i)[:1], T, B, nn.layerSize).cpu().numpy()
        f = _ws_array(nn, *_hook(nn, 1, i)[:1], T, B, nn.layerSize).cpu().numpy()
        b = _ws_array(nn, *_hook(nn, 2, i)[:1], T, B, nn.layerSize).cpu().numpy()
        assert np.array_equal(x.view(np.uint32), (f + b).view(np.uint32)), i


def test_every_colsum_path_and_clamp_was_reached(cuda):
    """The column-sum cases above reached the wide and the narrow path, both clamps of the wide path's rows per
    block, an interior one with remainder rows, and more than one column block."""
    missing = [k for k, v in REACHED.items() if not v]
    if missing and _sms(cuda) != H100_SMS:
        pytest.skip("plans not reachable on this device: %s" % missing)
    assert not missing, missing
