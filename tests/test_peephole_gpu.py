"""GPU tests of the peephole connections of the LSTM cell (ctcb_brnn_config.peephole = 1) on one H100.

The sweep alone in peephole mode (ctcb_lstm_sweep_peephole_f32), on every plan, and the peephole weight gradients
alone (ctcb_lstm_peephole_grad_f32) are tests/test_lstm_plans_gpu.py.  Here the whole net against
tests/net_oracle.Net (tests/net_check.py) with P drawn non-zero, and micro-batches, shards, graph
replay, forward-only probabilities, runNNet and checkpoints.  Each comparison prints its measured numbers as one JSON
line (pytest -s)."""
import json
import os
import pickle

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net

pytestmark = pytest.mark.gpu
COST_TOL, FWD_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-4


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
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make net c."""
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
    on = Net(D, K, H, N, c["T"], **_kwargs(c, reg))
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
        on = Net(D, K, c["H"], c["N"], c["T"], **_kwargs(c))
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
