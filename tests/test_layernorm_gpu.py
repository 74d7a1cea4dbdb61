"""GPU tests of layer normalisation (ctcb_brnn_config.layerNorm = 1) on one H100.

1. The kernels alone (ctcb_layernorm_forward_f32 / _backward_f32) against float64 of their own float32 inputs,
   element-wise, |x - x64| <= C u S with u = 2^-24 and S built from the magnitudes that make x:
     forward : the sums of a row have depth <= 8 (a thread's slots) + 5 (a warp) + 8 (the warps) + 4 (a float4), so
               the mean is off by at most ~25 u mean|z|; z - mu then carries that absolute error, scaled by rstd, and
               the rest is a few relative roundings: |xh - xh64| <= C u (mean|z| rstd + |xh|), |y - y64| <=
               C u (|gamma| (mean|z| rstd + |xh|) + |beta|), C_FWD = 64.  The same bound must reject a float32
               emulation of the one-pass variance E[z^2] - mu^2 on rows whose |mean| >> std.
     backward: from the kernel's own z, mu, rstd, gamma, g (xh64 = (z - mu) rstd in float64): dz against
               C u rstd (|gh| + mean|gh| + |xh| (mean|gh xh| + |b|)), b = mean(gh xh), C_FWD again; dgamma / dbeta
               sum over rows in chunks of rpp rows, then parts / 8 strided terms and 8: depth D = rpp + parts/8 + 8,
               |err| <= 2 (D + 4) u sum_r |g xh| (|g| for dbeta).
2. The whole net against tests/net_oracle.py (compared by tests/net_check.py): cost, every activation, and every
   gradient tensor against the oracle's back-propagation through the GPU's own activations (relative Frobenius <= 1e-4),
   for bi-, uni-directional, DNN, stacked, LSTM and dropout nets with mixed utterance lengths.
3. Consistency: micro-batches and shards, graph replay, forward-only probabilities, reruns; Adam and Nesterov; toFile /
   fromFile and the pair-count check; runNNet --layerNorm end to end; check_grad and a finite difference of beta.
Each comparison prints its measured errors as one JSON line (pytest -s)."""
import io
import json
import os
import pickle

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
C_FWD = 64.0
FWD_TOL, GRAD_TOL = 1e-4, 1e-4


def _ratio(err, bound):
    """max err / bound, NaN anywhere counting as infinitely far."""
    err, bound = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(bound, np.float64))
    if not np.all(np.isfinite(err)):
        return float("inf")
    if np.any(err[bound <= 0.0] != 0.0):
        return float("inf")
    pos = bound > 0.0
    return float(np.max(err[pos] / bound[pos])) if pos.any() else 0.0


# ------------------------------------------------------------------------------------------------ 1. the kernels
def _rows(R, H, rng):
    """Rows of mixed scale; a third with |mean| >> std (means 1000, -300, 100 with std 0.1), a few constant."""
    z = (rng.randn(R, H) * rng.uniform(0.1, 3.0, size=(R, 1)) + rng.randn(R, 1)).astype(np.float32)
    big = np.arange(0, R, 3)
    z[big] = (rng.choice([1000.0, -300.0, 100.0], size=(len(big), 1)) + 0.1 * rng.randn(len(big), H)).astype(np.float32)
    const = np.arange(1, R, 17)
    z[const] = np.float32(0.7)
    return z, big


def _fwd64(z, gamma, beta):
    z = z.astype(np.float64)
    mu = z.mean(axis=1, keepdims=True)
    var = ((z - mu) ** 2).mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + 1e-5)
    xh = (z - mu) * rstd
    y = np.maximum(gamma * xh + beta, 0.0)
    M = np.abs(z).mean(axis=1, keepdims=True)
    X = M * rstd + np.abs(xh)
    return mu, rstd, y, X


def _one_pass(z, gamma, beta):
    """float32 emulation of the one-pass variance E[z^2] - mu^2: what the bound must catch."""
    z = z.astype(np.float32)
    mu = z.mean(axis=1, dtype=np.float32, keepdims=True)
    ez2 = (z * z).mean(axis=1, dtype=np.float32, keepdims=True)
    with np.errstate(invalid="ignore"):
        rstd = np.float32(1.0) / np.sqrt(ez2 - mu * mu + np.float32(1e-5))
    return np.maximum(gamma.astype(np.float32) * ((z - mu) * rstd) + beta.astype(np.float32), np.float32(0.0))


def _ln_parts(R):
    rpp = max(8, -(-R // 1024))
    return rpp, -(-R // rpp)


@pytest.mark.parametrize("H,R", [(13, 1000), (64, 1000), (512, 1000), (1824, 1000), (2048, 1000), (64, 20000),
                                 (70, 333), (8192, 40), (3001, 1000), (4096, 1000), (1023, 1000), (8191, 40),
                                 (2048, 5000)])
def test_kernels_match_float64_of_their_inputs(H, R, cuda):
    torch = cuda
    from _ctcb import lib, check
    rng = np.random.RandomState(H + R)
    z, big = _rows(R, H, rng)
    gamma = (1.0 + 0.5 * rng.randn(1, H)).astype(np.float32)
    beta = (0.3 * rng.randn(1, H)).astype(np.float32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()        # noqa: E731
    dz, dg, db = dev(z), dev(gamma), dev(beta)
    y = torch.empty_like(dz)
    mu = torch.empty(R, dtype=torch.float32, device="cuda")
    rstd = torch.empty_like(mu)
    st = torch.cuda.current_stream().cuda_stream
    check(lib.ctcb_layernorm_forward_f32(dz.data_ptr(), y.data_ptr(), mu.data_ptr(), rstd.data_ptr(), dg.data_ptr(),
                                         db.data_ptr(), R, H, st))
    # forward-only (no statistics) and in place: the same bits
    y2 = torch.empty_like(dz)
    check(lib.ctcb_layernorm_forward_f32(dz.data_ptr(), y2.data_ptr(), None, None, dg.data_ptr(), db.data_ptr(), R, H, st))
    zin = dz.clone()
    check(lib.ctcb_layernorm_forward_f32(zin.data_ptr(), zin.data_ptr(), None, None, dg.data_ptr(), db.data_ptr(), R, H,
                                         st))
    assert np.array_equal(_bits(y), _bits(y2)) and np.array_equal(_bits(y), _bits(zin))
    mu64, rstd64, y64, X = _fwd64(z, gamma.astype(np.float64), beta.astype(np.float64))
    M = np.abs(z.astype(np.float64)).mean(axis=1, keepdims=True)
    bound_y = C_FWD * U32 * (np.abs(gamma) * X + np.abs(beta))
    r_y = _ratio(np.abs(y.cpu().numpy() - y64), bound_y)
    r_mu = _ratio(np.abs(mu.cpu().numpy()[:, None] - mu64), C_FWD * U32 * M)
    r_rstd = _ratio(np.abs(rstd.cpu().numpy()[:, None] - rstd64),
                    C_FWD * U32 * rstd64 * (1.0 + C_FWD * U32 * (M * rstd64) ** 2))
    one = np.abs(_one_pass(z, gamma, beta) - y64)
    r_one = _ratio(one[big], bound_y[big])

    # backward from the kernel's own inputs: g with zero rows (padded frames), gamma, z, its mu / rstd
    g = (rng.randn(R, H) * rng.uniform(0.01, 2.0, size=(R, 1))).astype(np.float32)
    g[2::11] = 0.0
    mu_g, rstd_g = mu.cpu().numpy().astype(np.float64)[:, None], rstd.cpu().numpy().astype(np.float64)[:, None]
    ws = torch.zeros(int(lib.ctcb_layernorm_workspace_bytes(R, H)), dtype=torch.uint8, device="cuda")
    prev_g, prev_b = (rng.randn(1, H) * 10).astype(np.float32), (rng.randn(1, H) * 10).astype(np.float32)
    out = {}
    for acc in (0, 1):
        d = dev(g)
        pg, pb = dev(prev_g), dev(prev_b)
        check(lib.ctcb_layernorm_backward_f32(d.data_ptr(), dz.data_ptr(), mu.data_ptr(), rstd.data_ptr(), dg.data_ptr(),
                                              pg.data_ptr(), pb.data_ptr(), R, H, acc, ws.data_ptr(), ws.numel(), st))
        out[acc] = (d.cpu().numpy(), pg.cpu().numpy(), pb.cpu().numpy())
    g64, gam = g.astype(np.float64), gamma.astype(np.float64)
    xh = (z.astype(np.float64) - mu_g) * rstd_g
    gh = g64 * gam
    a = gh.mean(axis=1, keepdims=True)
    b = (gh * xh).mean(axis=1, keepdims=True)
    dz64 = rstd_g * (gh - a - xh * b)
    bound_dz = C_FWD * U32 * rstd_g * (np.abs(gh) + np.abs(gh).mean(axis=1, keepdims=True) +
                                       np.abs(xh) * ((np.abs(gh * xh)).mean(axis=1, keepdims=True) + np.abs(b)))
    rpp, parts = _ln_parts(R)
    D = rpp + -(-parts // 8) + 8
    dgam64, dbet64 = (g64 * xh).sum(axis=0, keepdims=True), g64.sum(axis=0, keepdims=True)
    bg = 2 * (D + 4) * U32 * np.abs(g64 * xh).sum(axis=0, keepdims=True)
    bb = 2 * (D + 4) * U32 * np.abs(g64).sum(axis=0, keepdims=True)
    r_dz = max(_ratio(np.abs(out[acc][0] - dz64), bound_dz) for acc in (0, 1))
    assert np.array_equal(out[0][0], out[1][0])
    assert not out[0][0][2::11].view(np.uint32).any()     # zero delta rows stay +0.0, whatever the sign of gamma
    r_dg = _ratio(np.abs(out[0][1] - dgam64), bg)
    r_db = _ratio(np.abs(out[0][2] - dbet64), bb)
    r_dg_acc = _ratio(np.abs(out[1][1] - (dgam64 + prev_g)), bg + U32 * np.abs(dgam64 + prev_g))
    r_db_acc = _ratio(np.abs(out[1][2] - (dbet64 + prev_b)), bb + U32 * np.abs(dbet64 + prev_b))
    res = dict(y=r_y, mu=r_mu, rstd=r_rstd, one_pass_big_rows=r_one, dz=r_dz, dgamma=r_dg, dbeta=r_db,
               dgamma_acc=r_dg_acc, dbeta_acc=r_db_acc)
    print(json.dumps({"layernorm_kernels_H%d_R%d" % (H, R): res}))
    assert max(r_y, r_mu, r_rstd, r_dz, r_dg, r_db, r_dg_acc, r_db_acc) <= 1.0, res
    assert r_one > 1.0, "the bound does not catch the one-pass variance"
    # rerun: the same bytes
    d = dev(g)
    pg, pb = dev(prev_g), dev(prev_b)
    check(lib.ctcb_layernorm_backward_f32(d.data_ptr(), dz.data_ptr(), mu.data_ptr(), rstd.data_ptr(), dg.data_ptr(),
                                          pg.data_ptr(), pb.data_ptr(), R, H, 0, ws.data_ptr(), ws.numel(), st))
    assert np.array_equal(d.cpu().numpy().view(np.uint32), out[0][0].view(np.uint32))
    assert np.array_equal(pg.cpu().numpy().view(np.uint32), out[0][1].view(np.uint32))


# ------------------------------------------------------------------------------------------------ 2. the whole net
D_IN, K = 23, 17
NETS = {
    "bi_h64": dict(H=64, N=3, tl=2, k=1, T=30, B=6, L=8),
    "uni_h70": dict(H=70, N=3, tl=2, k=1, T=25, B=5, L=6, uni=True),
    "dnn_h64": dict(H=64, N=3, tl=0, k=0, T=20, B=5, L=6),
    "bi_stack2_h64": dict(H=64, N=4, tl=2, k=2, T=20, B=5, L=6),
    "lstm_bi_h64": dict(H=64, N=3, tl=2, k=1, T=20, B=5, L=6, cell="lstm"),
    "bi_dropout_h64": dict(H=64, N=3, tl=2, k=1, T=25, B=6, L=6, p=0.1),
    "bi_h512": dict(H=512, N=3, tl=2, k=1, T=12, B=4, L=4),
}


def _kwargs(c, reg=0.0):
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make net c."""
    return dict(temporalLayer=c["tl"] or -1, numTemporal=max(1, c["k"]), reg=reg, unidirectional=bool(c.get("uni")),
                cell=c.get("cell", "relu"), dropout=c.get("p", 0.0), layerNorm=True)


def _gpu_net(c, B, reg=0.0, train=True):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D_IN, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg))


def _ragged(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    rng = np.random.RandomState(seed)
    lens = [int(x) for x in rng.randint(max(1, int(0.5 * T)), T + 1, size=B)]
    lens[0] = T
    nlabs = [int(x) for x in rng.randint(1, L + 1, size=B)]
    return lens, recipes.synth_batch(D_IN, K, lens, nlabs, seed=33)


@pytest.mark.parametrize("name", list(NETS))
def test_layer_norm_net_matches_float64_oracle(name, cuda):
    c = NETS[name]
    lens, (datas, labelss) = _ragged(c)
    B, N = c["B"], c["N"]
    reg = 1e-3
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = Net(D_IN, K, c["H"], N, c["T"], **_kwargs(c, reg))
    on.initParams()
    assert nn.normedLayers() == on.normedLayers() and len(nn.normedLayers()) > 0
    for (w, b), (ow, ob) in zip(nn.stack, on.stack):        # the same draws, shapes and order; gamma 1, beta 0
        assert np.array_equal(w.cpu().numpy(), ow.astype(np.float32)) and tuple(b.shape) == ob.shape
        assert np.array_equal(b.cpu().numpy(), ob.astype(np.float32))
    rng = np.random.RandomState(3)                           # move gamma and beta off 1 and 0 on both sides
    for i in on.normedLayers():
        kk = on.ln_index(i)
        for t in range(2):
            v = (on.stack[kk][t] + 0.2 * rng.randn(*on.stack[kk][t].shape)).astype(np.float32)
            on.stack[kk][t] = v.astype(np.float64)
            nn.stack[kk][t].copy_(cuda.from_numpy(v))
    nn.costAndGradBatch(datas, labelss)
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    cost_err, fwd = r["cost_own"], max(r["fwd"]["X"])
    grad_err, grad_elem, plain = r["grad_given"], r["grad_given_elem"], r["grad_plain"]
    print(json.dumps({"layernorm_net_" + name: dict(cost=cost_err, fwd=fwd, grad_given_frob_max=max(grad_err),
                                                    grad_given_elem_max=max(grad_elem), grad_plain_frob_max=max(plain))}))
    assert cost_err <= FWD_TOL and fwd <= FWD_TOL
    assert max(grad_err) <= GRAD_TOL, grad_err


# ------------------------------------------------------------------------------------------------ 3. consistency
def _small(maxUtts, reg=0.0, uni=False, dropout=0.0, layerNorm=True, tl=2):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=tl, reg=reg, maxUtts=maxUtts, maxLabels=20,
                           unidirectional=uni, dropout=dropout, layerNorm=layerNorm)
    nn.initParams()
    return nn


def _batch8(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


@pytest.mark.parametrize("uni,dropout", [(False, 0.0), (True, 0.1)])
def test_micro_batches_and_two_shards_match_one_call(uni, dropout, cuda):
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    reg = 1e-2
    datas, labelss = _batch8()
    full = _small(8, reg, uni, dropout)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    g1 = full.grads_ext[:full.nparams + 4].cpu().numpy().astype(np.float64)
    split = _small(3, reg, uni, dropout)            # three micro-batches of 3, 3, 2
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 4].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):                           # two emulated shards, deferred L2 applied once to their sum
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4, reg, uni, dropout)
        nn.dropoutShard = (rank, 2)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    n_ln = 2 * 64 * len(full.normedLayers())
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    e_ln = max(_rel(g2[full.nparams - n_ln:-4], g1[full.nparams - n_ln:-4]),
               _rel(g3[full.nparams - n_ln:-4], g1[full.nparams - n_ln:-4]))
    print(json.dumps({"layernorm_accum_%s_p%g" % ("uni" if uni else "bi", dropout):
                      dict(micro=e_micro, shards=e_shard, ln_pairs=e_ln, cost=float(np.max(np.abs(c2 - c1))))}))
    assert np.allclose(c1, c2, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5 and e_ln < 1e-5
    assert g2[-4] == g3[-4] == g1[-4] == 8 and g1[-1] == g2[-1] == g3[-1] == 0


def test_l2_leaves_gamma_and_beta_alone(cuda):
    """reg > 0 adds reg * W to the weight matrices only: the gradient of the pairs is the same with and without it."""
    datas, labelss = _batch8()
    a, b = _small(8, 0.0), _small(8, 0.5)
    a.costAndGradBatch(datas, labelss)
    b.costAndGradBatch(datas, labelss)
    n_ln = 2 * 64 * len(a.normedLayers())
    ga, gb = a.grads.cpu().numpy(), b.grads.cpu().numpy()
    assert np.array_equal(ga[-n_ln:], gb[-n_ln:])
    assert not np.array_equal(ga[:64], gb[:64])


def _train(useGraphs, optimizer="nesterov", dropout=0.0, steps=5, uni=False, alpha=1e-3):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8, 1e-3, uni, dropout=dropout)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=alpha, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False, optimizer=optimizer)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn.params.cpu().numpy(), np.array(opt.costt), opt


@pytest.mark.parametrize("optimizer,dropout,uni", [("nesterov", 0.0, False), ("adam", 0.1, True),
                                                   ("nesterov", 0.1, False)])
def test_graph_replay_is_bit_identical_to_eager_steps(optimizer, dropout, uni, cuda):
    p_g, c_g, opt_g = _train(True, optimizer, dropout, uni=uni)
    p_e, c_e, opt_e = _train(False, optimizer, dropout, uni=uni)
    print(json.dumps({"layernorm_graph_%s_p%g_%s" % (optimizer, dropout, "uni" if uni else "bi"):
                      dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1 and len(opt_e._graphs) == 0
    assert np.array_equal(p_g, p_e) and np.array_equal(c_g, c_e)
    assert np.isfinite(p_g).all()


@pytest.mark.parametrize("optimizer,alpha", [("adam", 1e-3), ("nesterov", 1e-2)])
def test_optimisers_train_a_layer_norm_net(optimizer, alpha, cuda):
    """Twenty steps on one minibatch lower its cost."""
    _, costs, _ = _train(True, optimizer, steps=20, alpha=alpha)
    print(json.dumps({"layernorm_%s_costs" % optimizer: costs.tolist()}))
    assert np.isfinite(costs).all() and costs[-1] < 0.9 * costs[0]


def test_forward_only_probs_are_bit_identical_to_a_training_call(cuda):
    for name in ("bi_h64", "uni_h70", "dnn_h64", "lstm_bi_h64"):
        c = NETS[name]
        lens, (datas, labelss) = _ragged(c)
        np.random.seed(3)
        nn = _gpu_net(dict(c, p=0.0), c["B"])
        nn.initParams()
        batch = nn._batch.pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, want_probs=True)
        p_train = _bits(nn._probs_view(batch.B, batch.Tmax).clone())
        p_fwd = _bits(nn._forward_device(batch).clone())
        assert np.array_equal(p_train, p_fwd), name
        np.random.seed(3)
        inf = _gpu_net(dict(c, p=0.0), c["B"], train=False)
        inf.initParams()
        out = inf.forwardBatch(datas)
        probs = p_fwd.view(np.float32).reshape(batch.Tmax, batch.B, K)
        for u, d in enumerate(datas):
            assert np.array_equal(out[u], probs[:d.shape[1], u, :].T), name


def test_two_runs_give_the_same_bytes(cuda):
    datas, labelss = _batch8()
    outs = []
    for _ in range(2):
        nn = _small(8, 1e-3, dropout=0.1)
        nn.costAndGradBatch(datas, labelss)
        first = _bits(nn.grads_ext).copy()
        nn.costAndGradBatch(datas, labelss)
        assert np.array_equal(first, _bits(nn.grads_ext))
        outs.append(first)
    assert np.array_equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ checkpoints, runNNet
def test_checkpoints_round_trip_and_refuse_a_net_without_pairs(cuda):
    import sgd
    datas, labelss = _batch8()
    a = _small(8)
    for w, b in a.stack[-2:]:
        w.add_(0.25)
        b.add_(-0.5)
    f = io.BytesIO()
    a.toFile(f)
    f.seek(0)
    b = _small(8)
    b.fromFile(f)
    assert np.array_equal(a.params.cpu().numpy(), b.params.cpu().numpy())
    plain = _small(8, layerNorm=False)
    f = io.BytesIO()
    plain.toFile(f)
    f.seek(0)
    with pytest.raises(ValueError, match="pairs"):
        b.fromFile(f)
    # the optimiser state carries the pairs too, and SGD.fromFile checks its count the same way
    opt = sgd.SGD(b, 60, verbose=False)
    f = io.BytesIO()
    opt.toFile(f)
    assert len(pickle.loads(f.getvalue())[3]) == len(b.stack)
    f.seek(0)
    sgd.SGD(_small(8), 60, verbose=False).fromFile(f)
    f = io.BytesIO()
    sgd.SGD(plain, 60, verbose=False).toFile(f)
    f.seek(0)
    with pytest.raises(ValueError, match="pairs"):
        sgd.SGD(b, 60, verbose=False).fromFile(f)
    del datas, labelss


def test_run_nnet_trains_resumes_and_tests_a_layer_norm_net(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--layerNorm", "--epochs", "1",
            "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16", "--rawDim", "20",
            "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1",
            "--runDir", str(tmp_path / "runs"), "--quiet"]
    _, net = runNNet.run(args)
    assert net.layerNorm and net.normedLayers() == [1, 3] and len(net.stack) == 4 + 2 + 2
    assert not np.array_equal(net.stack[6][0].cpu().numpy(), np.ones((64, 1), np.float32))     # gamma trained
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["layerNorm"] is True
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.layerNorm and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert tnet.layerNorm and not tnet.train
    assert np.array_equal(tnet.params.cpu().numpy(), p_epoch0)
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16


# ------------------------------------------------------------------------------------------------ finite differences
def test_check_grad_and_beta_by_finite_differences(cuda):
    """NNet.check_grad (forward differences in fp32, as test_brnn_gpu.py) covers the first tensor of each pair, gamma
    included; beta by central differences here.  gamma and beta are moved off 1 and 0 first."""
    import nnets.brnnet as rnnet
    datas, labelss = recipes.synth_batch(6, 5, [12], [3], seed=4)
    np.random.seed(8)
    nn = rnnet.NNet(6, 5, 8, 2, 12, temporalLayer=1, layerNorm=True)
    nn.initParams()
    rng = np.random.RandomState(1)
    gamma, beta = nn.stack[-1]
    gamma.add_(nn._torch.from_numpy((0.3 * rng.randn(8, 1)).astype(np.float32)).cuda())
    beta.add_(nn._torch.from_numpy((0.3 * rng.randn(8, 1)).astype(np.float32)).cuda())
    pairs = nn.check_grad(datas[0], labelss[0], epsilon=1e-3, maxChecks=2, verbose=False)
    ana = np.array([p[0] for p in pairs]); num = np.array([p[1] for p in pairs])
    assert len(pairs) == 5 * 4 + 2                  # W1, W2, W3, Wtf, Wtb (2 x 2 each), gamma (2 x 1)
    assert np.abs(ana - num).max() < 0.05 * max(1.0, np.abs(ana).max())
    cost, grad, _ = nn.costAndGrad(datas[0], labelss[0])
    dbeta = grad[-1][1].cpu().numpy().copy()
    eps = 1e-2
    errs = []
    for j in range(8):
        beta[j, 0] += eps
        cp, _, _ = nn.costAndGrad(datas[0], labelss[0])
        beta[j, 0] -= 2 * eps
        cm, _, _ = nn.costAndGrad(datas[0], labelss[0])
        beta[j, 0] += eps
        errs.append(float(abs((cp - cm) / (2 * eps) - dbeta[j, 0])))
    print(json.dumps({"layernorm_fd_beta": dict(max_err=max(errs), max_dbeta=float(np.abs(dbeta).max()))}))
    assert max(errs) < 0.05 * max(1.0, float(np.abs(dbeta).max()))
