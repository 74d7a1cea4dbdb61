"""GPU tests of the peephole connections of the LSTM cell (ctcb_brnn_config.peephole = 1) on one H100.

The sweep alone (ctcb_lstm_sweep_peephole_f32) against the float64 recurrence of tests/peephole_oracle.py computed
from the kernel's own float32 inputs, element-wise, with the bound of tests/test_lstm_gpu.py: |x - x64| <= C u S,
u = 2^-24, S the sum of the magnitudes of the terms that make x, the float64 of the step computed from the GPU's own state of the
step before (S = 1 + |pre| + |U| |h_prev| + |p| |c_prev| for the i and f gates, + |p_o| |c_t| for o; |f c_prev| + |i g|
for c; |o| for h), C = 8; dz, which carries the whole dc term from step to step inside the kernel, against the float64
BPTT of the GPU's own forward activations with S = max(1, max |dz64|), C = 32.  The peephole weight gradients
(ctcb_lstm_peephole_grad_f32) against float64 of their inputs with a bound derived below.  Then the whole net
against peephole_oracle.PeepholeNet (tests/net_check.py) with P drawn non-zero, and micro-batches, shards, graph
replay, forward-only probabilities, runNNet and checkpoints.  Each comparison prints its measured numbers as one JSON
line (pytest -s)."""
import ctypes
import json
import os
import pickle

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from peephole_oracle import PeepholeNet, lstm_direction_bptt

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
C_FWD, C_BPTT = 8.0, 32.0
COST_TOL, FWD_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-4


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def _p(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------ the sweep alone
SWEEPS = [(H, uni, B, T) for H in (64, 70, 512, 1024) for uni in (False, True) for B, T in ((1, 1), (13, 9))] + \
    [(1024, False, 128, 5), (70, True, 128, 4), (512, False, 128, 3)]


@pytest.mark.parametrize("H,uni,B,T", SWEEPS)
def test_peephole_sweep_matches_float64(H, uni, B, T, cuda):
    torch = cuda
    from _ctcb import lib, check
    ndir = 1 if uni else 2
    G = ndir * 4 * H
    plan = (ctypes.c_int32 * 2)()
    check(lib.ctcb_debug_lstm_plan(H, B, ndir, plan))
    rng = np.random.RandomState(H + B + T + 1)
    lens = rng.randint(1, T + 1, size=B).astype(np.int32)
    lens[0] = T
    pre = rng.uniform(-1.5, 1.5, (T, B, G)).astype(np.float32)
    s = 1.5 / np.sqrt(H)
    Us = [rng.uniform(-s, s, (4 * H, H)).astype(np.float32) for _ in range(ndir)]
    Ps = [rng.uniform(-0.5, 0.5, (3, H)).astype(np.float32) for _ in range(ndir)]
    dh = rng.randn(T, B, H).astype(np.float32)
    dev = torch.device("cuda")
    d_pre = torch.from_numpy(pre).to(dev)
    d_U = [torch.from_numpy(u).to(dev) for u in Us]
    d_P = [torch.from_numpy(x).to(dev) for x in Ps]
    d_h = [torch.full((T, B, H), float("nan"), device=dev) for _ in range(ndir)]
    d_c = [torch.full((T, B, H), float("nan"), device=dev) for _ in range(ndir)]
    d_dh = torch.from_numpy(dh).to(dev)
    d_dz = torch.full((T, B, G), float("nan"), device=dev)
    d_len = torch.from_numpy(lens).to(dev)
    ws = lib.ctcb_lstm_sweep_workspace_bytes(H, B)
    scratch = torch.zeros(ws, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    Ub, Pb, hB, cB = (None, None, None, None) if uni else (d_U[1], d_P[1], d_h[1], d_c[1])
    check(lib.ctcb_lstm_sweep_peephole_f32(0, T, B, H, _p(d_len), _p(d_pre), _p(d_U[0]), _p(Ub), _p(d_P[0]), _p(Pb),
                                           _p(d_h[0]), _p(hB), _p(d_c[0]), _p(cB), None, None, _p(scratch), ws, st))
    check(lib.ctcb_lstm_sweep_peephole_f32(1, T, B, H, _p(d_len), _p(d_pre), _p(d_U[0]), _p(Ub), _p(d_P[0]), _p(Pb),
                                           None, None, _p(d_c[0]), _p(cB), _p(d_dh), _p(d_dz), _p(scratch), ws, st))
    torch.cuda.synchronize()
    assert int(scratch[:4].view(torch.int32).item()) == 0
    gates = d_pre.cpu().numpy().astype(np.float64)
    hs = [x.cpu().numpy().astype(np.float64) for x in d_h]
    cs = [x.cpu().numpy().astype(np.float64) for x in d_c]
    dz = d_dz.cpu().numpy().astype(np.float64)
    ratio = dict(gates=0.0, c=0.0, h=0.0, dz=0.0)
    for u in range(B):
        Tu = int(lens[u])
        for d in range(ndir):
            blk = slice(d * 4 * H, (d + 1) * 4 * H)
            for arr in (gates[Tu:, u, blk], hs[d][Tu:, u], cs[d][Tu:, u], dz[Tu:, u, blk]):
                assert not np.any(arr), "padded frame not 0"
            U, P = Us[d].astype(np.float64), Ps[d].astype(np.float64)
            g, c, h = gates[:Tu, u, blk].T, cs[d][:Tu, u].T, hs[d][:Tu, u].T
            pz = pre[:Tu, u, blk].T.astype(np.float64)
            for t in range(Tu):
                tp = t + 1 if d == 1 else t - 1
                hp = h[:, tp] if 0 <= tp < Tu else np.zeros(H)
                cp = c[:, tp] if 0 <= tp < Tu else np.zeros(H)
                z = pz[:, t] + U.dot(hp)
                Sz = 1.0 + np.abs(pz[:, t]) + np.abs(U).dot(np.abs(hp))
                i64 = _sig(z[:H] + P[0] * cp)
                f64 = _sig(z[H:2 * H] + P[1] * cp)
                g64 = np.tanh(z[2 * H:3 * H])
                o64 = _sig(z[3 * H:] + P[2] * c[:, t])     # from the GPU's own c_t
                S = Sz + np.concatenate([np.abs(P[0] * cp), np.abs(P[1] * cp), np.zeros(H), np.abs(P[2] * c[:, t])])
                a64 = np.concatenate([i64, f64, g64, o64])
                ratio["gates"] = max(ratio["gates"], float(np.max(np.abs(g[:, t] - a64) / (U32 * S))))
                i_, f_, g_, o_ = g[:H, t], g[H:2 * H, t], g[2 * H:3 * H, t], g[3 * H:, t]
                c64 = f_ * cp + i_ * g_
                Sc = np.abs(f_ * cp) + np.abs(i_ * g_) + 1e-30
                ratio["c"] = max(ratio["c"], float(np.max(np.abs(c[:, t] - c64) / (U32 * Sc))))
                h64 = o_ * np.tanh(c[:, t])
                ratio["h"] = max(ratio["h"], float(np.max(np.abs(h[:, t] - h64) / (U32 * (np.abs(o_) + 1e-30)))))
            dz64, _, _ = lstm_direction_bptt(dh[:Tu, u].T.astype(np.float64), g, c, h, U, reverse=(d == 1), peephole=P)
            S = max(1.0, float(np.max(np.abs(dz64))))
            ratio["dz"] = max(ratio["dz"], float(np.max(np.abs(dz[:Tu, u, blk].T - dz64)) / (U32 * S)))
    print(json.dumps({"peephole_sweep_H%d_%s_B%d_T%d" % (H, "uni" if uni else "bi", B, T):
                      dict(plan_KI=plan[0], parts=plan[1], **ratio)}))
    assert ratio["gates"] <= C_FWD and ratio["c"] <= C_FWD and ratio["h"] <= C_FWD
    assert ratio["dz"] <= C_BPTT


# ------------------------------------------------------------------------------------------------ dP alone
@pytest.mark.parametrize("T,B,H,ndir", [(1, 3, 64, 2), (9, 13, 70, 1), (37, 5, 512, 2), (300, 8, 1024, 2)])
def test_peephole_grad_matches_float64(T, B, H, ndir, cuda):
    """dP against float64 of the same float32 dz and c.  Each output is a sum of n = T B products, each product exact
    to u in float32 and the sum of fixed chunks of 1024 rows (8 interleaved partial sums of 128 products each, combined
    in a tree of 8, then the chunks in order): a recursive sum of m terms errs by at most (m - 1) u sum |terms|, so the
    bound is (128 + 8 + ceil(n / 1024) + 1) u sum |dz c'|.  A rerun is bit-identical, and accumulate adds."""
    torch = cuda
    from _ctcb import lib, check
    rng = np.random.RandomState(T + B + H)
    G = ndir * 4 * H
    lens = rng.randint(1, T + 1, size=B)
    lens[0] = T
    mask = (np.arange(T)[:, None] < lens[None, :]).astype(np.float32)        # [T][B]
    dz = (rng.randn(T, B, G) * mask[:, :, None]).astype(np.float32)
    cs = [(rng.randn(T, B, H) * mask[:, :, None]).astype(np.float32) for _ in range(ndir)]
    dev = torch.device("cuda")
    d_dz = torch.from_numpy(dz).to(dev)
    d_c = [torch.from_numpy(c).to(dev) for c in cs]
    d_dP = [torch.full((3, H), float("nan"), device=dev) for _ in range(ndir)]
    nbytes = lib.ctcb_lstm_peephole_grad_workspace_bytes(T, B, H, ndir)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    cB, dPb = (None, None) if ndir == 1 else (d_c[1], d_dP[1])

    def run(acc):
        check(lib.ctcb_lstm_peephole_grad_f32(T, B, H, _p(d_dz), _p(d_c[0]), _p(cB), _p(d_dP[0]), _p(dPb), acc, _p(ws),
                                              nbytes, st))
        torch.cuda.synchronize()
        return [x.cpu().numpy().copy() for x in d_dP]

    first = run(0)
    again = run(0)
    twice = run(1)
    n = T * B
    K = 128 + 8 + (n + 1023) // 1024 + 1
    worst = 0.0
    for d in range(ndir):
        blk = dz[:, :, d * 4 * H:(d + 1) * 4 * H].astype(np.float64)
        c = cs[d].astype(np.float64)
        cprev = np.zeros_like(c)
        if d == 0:
            cprev[1:] = c[:-1]
        else:
            cprev[:-1] = c[1:]
        terms = [blk[:, :, :H] * cprev, blk[:, :, H:2 * H] * cprev, blk[:, :, 3 * H:] * c]
        want = np.stack([x.sum(axis=(0, 1)) for x in terms])
        S = np.stack([np.abs(x).sum(axis=(0, 1)) for x in terms]) + 1e-30
        worst = max(worst, float(np.max(np.abs(first[d] - want) / (K * U32 * S))))
        assert np.array_equal(first[d].view(np.uint32), again[d].view(np.uint32))
        assert np.array_equal(twice[d], first[d] + first[d])       # x + x is exact
    print(json.dumps({"peephole_grad_T%d_B%d_H%d_%s" % (T, B, H, "bi" if ndir == 2 else "uni"):
                      dict(ratio_to_bound=worst, bound_C=K)}))
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------ the whole net
D, K = 23, 17
NETS = {
    "h64_bi_k1": dict(H=64, N=3, tl=2, k=1, T=30, B=6, L=8),
    "h70_uni_k2_ragged": dict(H=70, N=4, tl=2, k=2, T=25, B=5, L=6, uni=True, ragged=True),
    "h64_bi_k2_ragged_ln_drop": dict(H=64, N=4, tl=2, k=2, T=20, B=7, L=6, ragged=True, ln=True, p=0.3),
    "h512_bi_k1_sub_below": dict(H=512, N=3, tl=2, k=1, T=24, B=4, L=4, sub=(2, 1)),
    "h64_uni_k1_sub_above": dict(H=64, N=3, tl=1, k=1, T=21, B=5, L=4, uni=True, ragged=True, sub=(3, 2)),
    "h1024_bi_k1": dict(H=1024, N=2, tl=1, k=1, T=10, B=3, L=4),
    "h64_bi_k1_T1": dict(H=64, N=3, tl=1, k=1, T=1, B=3, L=1),
}


def _kwargs(c, reg=0.0):
    """The keyword arguments of nnets.brnnet.NNet and peephole_oracle.PeepholeNet that make net c."""
    k, L = c.get("sub", (1, 1))
    return dict(temporalLayer=c["tl"], numTemporal=c["k"], reg=reg, unidirectional=bool(c.get("uni")), cell="lstm",
                peephole=True, layerNorm=bool(c.get("ln")), dropout=c.get("p", 0.0), dropoutSeed=5, subsample=k,
                subsampleLayer=L)


def _gpu_net(c, B, reg=0.0, train=True):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg))


def _batch(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    k = c.get("sub", (1, 1))[0]
    if c.get("ragged"):
        rng = np.random.RandomState(seed)
        lens = [int(x) for x in rng.randint(max(1, int(0.5 * T)), T + 1, size=B)]
        lens[0] = T
        nlabs = [min(int(x), -(-n // k)) for x, n in zip(rng.randint(1, L + 1, size=B), lens)]
    else:
        lens, nlabs = [T] * B, [min(L, -(-T // k))] * B
    return lens, recipes.synth_batch(D, K, lens, nlabs, seed=33)


def _draw_p(stack, nn, seed=8):
    """P of every direction of every LSTM layer uniform in (-0.5, 0.5), the same float32 in both nets."""
    rng = np.random.RandomState(seed)
    n = nn.peepholeEntries()
    for w, _ in stack[len(stack) - n:]:
        x = rng.uniform(-0.5, 0.5, tuple(w.shape)).astype(np.float32)
        yield w, x


def _set_p(nn, on, seed=8):
    import torch
    for (w, x), (ow, _) in zip(_draw_p(nn.stack, nn, seed), on.stack[len(on.stack) - nn.peepholeEntries():]):
        w.copy_(torch.from_numpy(x))
        ow[...] = x


@pytest.mark.parametrize("name", list(NETS))
def test_peephole_net_matches_float64_oracle(name, cuda):
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    B, H, N = c["B"], c["H"], c["N"]
    reg = 1e-3
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = PeepholeNet(D, K, H, N, c["T"], **_kwargs(c, reg))
    on.initParams()
    for (w, b), (ow, ob) in zip(nn.stack, on.stack):        # the same draws, shapes and order, P = 0
        assert np.array_equal(w.cpu().numpy(), ow.astype(np.float32)) and tuple(b.shape) == ob.shape
    assert nn.peepholeEntries() == c["k"] * (1 if c.get("uni") else 2)
    _set_p(nn, on)
    if nn.dropout:
        nn.dropoutStep.fill_(3)
        on.dropoutStep = 3
    nn.costAndGradBatch(datas, labelss)
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    fwd = dict(logits=r["fwd"]["X"][N], gates=r["fwd"]["gates"], c=r["fwd"]["c"], h=r["fwd"]["h"])
    grad_err, grad_elem = r["grad_given"], r["grad_given_elem"]
    n = nn.peepholeEntries()
    p_err = [grad_err[-2 * n + 2 * x] for x in range(n)]
    dummies = [g[1] for g in nn.grad[len(nn.grad) - n:]]
    print(json.dumps({"peephole_net_" + name: dict(cost=r["cost_own"], fwd=fwd, grad_given_frob_max=max(grad_err),
                                                   grad_given_elem_max=max(grad_elem), dP_frob=p_err)}))
    assert all(float(d.abs().max()) == 0.0 for d in dummies)
    assert min(float(g[0].abs().max()) for g in nn.grad[len(nn.grad) - n:]) > 0.0
    assert r["cost_own"] <= COST_TOL
    assert max(fwd.values()) <= FWD_TOL, fwd
    assert max(grad_err) <= GRAD_TOL, grad_err


def test_forward_only_probs_are_bit_identical_to_a_training_call(cuda):
    for name in ("h64_bi_k2_ragged_ln_drop", "h70_uni_k2_ragged", "h64_uni_k1_sub_above"):
        c = dict(NETS[name], p=0.0)
        lens, (datas, labelss) = _batch(c)
        np.random.seed(3)
        nn = _gpu_net(c, c["B"])
        nn.initParams()
        on = PeepholeNet(D, K, c["H"], c["N"], c["T"], **_kwargs(c))
        np.random.seed(3)
        on.initParams()
        _set_p(nn, on)
        batch = nn._batch.pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, want_probs=True)
        p_train = _bits(nn._probs_view(batch.B, nn.frames(batch.Tmax)).clone())
        p_fwd = _bits(nn._forward_device(batch).clone())
        assert np.array_equal(p_train, p_fwd), name
        np.random.seed(3)
        inf = _gpu_net(c, c["B"], train=False)
        inf.initParams()
        inf.params.copy_(nn.params)
        out = inf.forwardBatch(datas)
        probs = p_fwd.view(np.float32).reshape(nn.frames(batch.Tmax), batch.B, K)
        for u, d in enumerate(datas):
            assert np.array_equal(out[u], probs[:nn.frames(d.shape[1]), u, :].T)


# ------------------------------------------------------------------------------------------------ accumulation
def _small(maxUtts, reg=0.0, uni=False, k=2, dropout=0.0, peephole=True):
    import nnets.brnnet
    import torch
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20, numTemporal=k,
                           unidirectional=uni, cell="lstm", dropout=dropout, peephole=peephole)
    nn.initParams()
    if peephole:
        for w, x in _draw_p(nn.stack, nn, 6):
            w.copy_(torch.from_numpy(x))
    return nn


def _ragged(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


@pytest.mark.parametrize("uni", [False, True])
def test_micro_batches_and_two_shards_match_one_call(uni, cuda):
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    reg = 1e-2
    datas, labelss = _ragged()
    full = _small(8, reg, uni)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    g1 = full.grads_ext[:full.nparams + 4].cpu().numpy().astype(np.float64)
    split = _small(3, reg, uni)                     # three micro-batches of 3, 3, 2
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 4].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):                           # two emulated shards, deferred L2 applied once to their sum
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4, reg, uni)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    n = full.peepholeEntries()
    P = np.concatenate([full.grad[len(full.grad) - n + x][0].cpu().numpy().ravel() for x in range(n)])
    offs = [full.grad[len(full.grad) - n + x][0].data_ptr() - full.grads.data_ptr() for x in range(n)]
    sl = np.concatenate([np.arange(o // 4, o // 4 + 3 * 64) for o in offs])
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    p_micro, p_shard = _rel(g2[sl], P), _rel(g3[sl], P)
    print(json.dumps({"peephole_accum_%s" % ("uni" if uni else "bi"): dict(micro=e_micro, shards=e_shard,
                                                                            dP_micro=p_micro,
                                                                            dP_shards=p_shard)}))
    assert np.allclose(c1, c2, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5 and p_micro < 1e-5 and p_shard < 1e-5
    assert g2[-4] == g3[-4] == g1[-4] == 8 and g1[-1] == g2[-1] == g3[-1] == 0


def _train(useGraphs, optimizer="nesterov", steps=5, uni=False):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8, 1e-3, uni)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False, optimizer=optimizer)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn, np.array(opt.costt), opt


@pytest.mark.parametrize("optimizer,uni", [("nesterov", False), ("adam", True)])
def test_graph_replay_is_bit_identical_to_eager_steps(optimizer, uni, cuda):
    nn_g, c_g, opt_g = _train(True, optimizer, uni=uni)
    nn_e, c_e, opt_e = _train(False, optimizer, uni=uni)
    p_g, p_e = nn_g.params.cpu().numpy(), nn_e.params.cpu().numpy()
    n = nn_g.peepholeEntries()
    moved = [float(np.abs(w.cpu().numpy() - x).max()) for (w, _), (_, x) in
             zip(nn_g.stack[len(nn_g.stack) - n:], _draw_p(nn_g.stack, nn_g, 6))]
    print(json.dumps({"peephole_graph_%s_%s" % (optimizer, "uni" if uni else "bi"):
                      dict(graphs=len(opt_g._graphs), costs=c_g.tolist(), P_moved=moved)}))
    assert len(opt_g._graphs) >= 1 and len(opt_e._graphs) == 0
    assert np.array_equal(p_g, p_e) and np.array_equal(c_g, c_e)
    assert np.isfinite(p_g).all() and min(moved) > 0.0


# ------------------------------------------------------------------------------------------------ Python surface
def test_peepholes_need_the_lstm_cell(cuda):
    import nnets.brnnet as brnnet
    import nnets.rnnet as rnnet
    with pytest.raises(ValueError, match="peephole=True needs cell='lstm'; cell is 'relu'"):
        brnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, peephole=True)
    with pytest.raises(ValueError, match="peephole"):
        rnnet.NNet(13, 11, 64, 3, 20, temporalLayer=2, peephole=True)
    nn = brnnet.NNet(13, 11, 64, 3, 20, temporalLayer=-1, cell="lstm", peephole=True)   # no temporal layer: nothing
    nn.initParams()
    assert nn.peepholeEntries() == 0 and len(nn.stack) == 4


def test_checkpoints_round_trip_and_refuse_the_other_setting(cuda, tmp_path):
    import io
    import sgd
    on = _small(4)
    off = _small(4, peephole=False)
    buf = io.BytesIO()
    on.toFile(buf)
    buf.seek(0)
    back = _small(4)
    back.params.zero_()
    back.fromFile(buf)
    assert np.array_equal(back.params.cpu().numpy(), on.params.cpu().numpy())
    for src, dst, text in ((off, on, "has 18 tensors where this net (cell='lstm', peephole=True) has 26: a checkpoint "
                                     "of an LSTM net without peephole"),
                           (on, off, "has 26 tensors where this net (cell='lstm', peephole=False) has 18: a checkpoint "
                                     "of an LSTM net with peephole")):
        buf = io.BytesIO()
        src.toFile(buf)
        buf.seek(0)
        with pytest.raises(ValueError, match=text.replace("(", r"\(").replace(")", r"\)")):
            dst.fromFile(buf)
        o_src = sgd.SGD(src, 60, alpha=1e-3, verbose=False)
        o_dst = sgd.SGD(dst, 60, alpha=1e-3, verbose=False)
        buf = io.BytesIO()
        o_src.toFile(buf)
        buf.seek(0)
        with pytest.raises(ValueError, match="optimiser state"):
            o_dst.fromFile(buf)


def test_check_grad_covers_the_peepholes(cuda):
    """check_grad probes every [w, b]'s w, P included: with eps = 1e-2 in float32 its forward differences of P agree
    with the analytic gradient."""
    import nnets.brnnet as brnnet
    import torch
    datas, labelss = recipes.synth_batch(13, 11, [30], [6], seed=2)
    np.random.seed(5)
    nn = brnnet.NNet(13, 11, 16, 3, 30, temporalLayer=2, cell="lstm", peephole=True, maxLabels=6)
    nn.initParams()
    for w, x in _draw_p(nn.stack, nn, 2):
        w.copy_(torch.from_numpy(x))
    out = nn.check_grad(datas[0], labelss[0], epsilon=1e-2, maxChecks=4, verbose=False)
    n_before = sum(min(w.shape[0], 4) * min(w.shape[1], 4) for w, _ in nn.stack[:-2])
    pairs = np.array(out[n_before:n_before + 12])           # the forward direction's P: 3 x 4 probes
    err = np.abs(pairs[:, 0] - pairs[:, 1]) / np.maximum(np.abs(pairs[:, 1]), 5e-2)
    print(json.dumps({"peephole_check_grad": dict(probes=len(out), P_rel_err_max=float(err.max()))}))
    assert len(out) == n_before + 2 * 12
    assert float(err.max()) < 0.1


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests_a_peephole_net(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--cell", "lstm", "--peephole",
            "--epochs", "1", "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16", "--rawDim",
            "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1",
            "--runDir", str(tmp_path / "runs"), "--quiet"]
    _, net = runNNet.run(args)
    assert net.peephole and tuple(net.stack[-2][0].shape) == (3, 64) and len(net.stack) == 8
    assert float(net.stack[-2][0].abs().max()) > 0.0         # P trained away from 0
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["peephole"] is True
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.peephole and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert tnet.peephole and not tnet.train
    assert np.array_equal(tnet.params.cpu().numpy(), p_epoch0)
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16
    # an LSTM net without peepholes cannot load the checkpoint
    import nnets.brnnet as brnnet
    plain = brnnet.NNet(16, 9, 64, 3, 40, temporalLayer=2, train=False, cell="lstm")
    plain.initParams()
    with open(os.path.join(run_dir, "params.pk"), "rb") as fid:
        pickle.load(fid)
        with pytest.raises(ValueError, match="peephole"):
            plain.fromFile(fid)
