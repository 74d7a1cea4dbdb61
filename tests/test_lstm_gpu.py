"""GPU tests of the LSTM cell (ctcb_brnn_config.cell = 1) on one H100.

The sweep alone, on every plan, is tests/test_lstm_plans_gpu.py.  Here the whole net against net_oracle.Net
(tests/net_check.py): per-utterance cost,
logits, gates, c and h of every LSTM layer relative to their largest magnitude (<= 1e-4), every gradient tensor against
the oracle's back-propagation through the GPU's own activations (relative Frobenius <= 1e-4, and the largest
element-wise error relative to the tensor's largest magnitude printed). Then micro-batches, two emulated shards, graph
replay, forward-only probabilities, dropout on the ReLU layers, Adam, runNNet end to end and a width the device cannot
hold. Each comparison prints its measured errors as one JSON line (pytest -s)."""
import ctypes
import json
import os

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel, workspace_activations
from net_oracle import Net

pytestmark = pytest.mark.gpu
COST_TOL, FWD_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-4


# ------------------------------------------------------------------------------------------------ the whole net
D, K = 23, 17
NETS = {
    "h64_bi_k1": dict(H=64, N=3, tl=2, k=1, T=30, B=6, L=8),
    "h70_uni_k2_ragged": dict(H=70, N=4, tl=2, k=2, T=25, B=5, L=6, uni=True, ragged=True),
    "h64_bi_k3_ragged": dict(H=64, N=5, tl=2, k=3, T=20, B=7, L=6, ragged=True),
    "h512_bi_k2": dict(H=512, N=3, tl=1, k=2, T=12, B=4, L=4),
    "h1024_uni_k1": dict(H=1024, N=2, tl=1, k=1, T=10, B=3, L=4, uni=True),
    "h64_bi_k2_T1": dict(H=64, N=3, tl=1, k=2, T=1, B=3, L=1),
}


def _kwargs(c, reg=0.0):
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make net c."""
    return dict(temporalLayer=c["tl"], numTemporal=c["k"], reg=reg, unidirectional=bool(c.get("uni")), cell="lstm")


def _gpu_net(c, B, reg=0.0, train=True):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg))


def _batch(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    if c.get("ragged"):
        rng = np.random.RandomState(seed)
        lens = [int(x) for x in rng.randint(max(1, int(0.5 * T)), T + 1, size=B)]
        lens[0] = T
        nlabs = [int(x) for x in rng.randint(1, L + 1, size=B)]
    else:
        lens, nlabs = [T] * B, [min(L, T)] * B
    return lens, recipes.synth_batch(D, K, lens, nlabs, seed=33)


@pytest.mark.parametrize("name", list(NETS))
def test_lstm_net_matches_float64_oracle(name, cuda):
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    B, H, N, tl, k = c["B"], c["H"], c["N"], c["tl"], c["k"]
    uni = bool(c.get("uni"))
    reg = 1e-3
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = Net(D, K, H, N, c["T"], **_kwargs(c, reg))
    on.initParams()
    for (w, b), (ow, ob) in zip(nn.stack, on.stack):        # the same draws, shapes and order
        assert np.array_equal(w.cpu().numpy(), ow.astype(np.float32)) and tuple(b.shape) == ob.shape
    nn.costAndGradBatch(datas, labelss)
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    cost_err = r["cost_own"]
    acts = r["acts"]
    for u in range(B):                      # padded frames of every LSTM buffer are exactly 0
        for i in range(tl, tl + k):
            for what in (0, 1, 4) + (() if uni else (2, 5)):
                assert not np.any(acts[what, i][lens[u]:, u]), "padded frame not 0"
    fwd = dict(logits=r["fwd"]["X"][N], gates=r["fwd"]["gates"], c=r["fwd"]["c"], h=r["fwd"]["h"])
    grad_err, grad_elem, plain = r["grad_given"], r["grad_given_elem"], r["grad_plain"]
    print(json.dumps({"lstm_net_" + name: dict(cost=cost_err, fwd=fwd, grad_given_frob_max=max(grad_err),
                                               grad_given_elem_max=max(grad_elem), grad_plain_frob_max=max(plain))}))
    assert cost_err <= COST_TOL
    assert max(fwd.values()) <= FWD_TOL, fwd
    assert max(grad_err) <= GRAD_TOL and max(grad_elem) <= GRAD_TOL, (grad_err, grad_elem)
    assert max(plain) <= GRAD_TOL, plain      # no clip or ReLU kink inside the cell: no mask flips to allow for


def test_forward_only_probs_are_bit_identical_to_a_training_call(cuda):
    for name in ("h64_bi_k3_ragged", "h70_uni_k2_ragged"):
        c = NETS[name]
        lens, (datas, labelss) = _batch(c)
        np.random.seed(3)
        nn = _gpu_net(c, c["B"])
        nn.initParams()
        batch = nn._batch.pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, want_probs=True)
        p_train = _bits(nn._probs_view(batch.B, batch.Tmax).clone())
        p_fwd = _bits(nn._forward_device(batch).clone())
        assert np.array_equal(p_train, p_fwd), name
        np.random.seed(3)
        inf = _gpu_net(c, c["B"], train=False)
        inf.initParams()
        out = inf.forwardBatch(datas)
        probs = p_fwd.view(np.float32).reshape(batch.Tmax, batch.B, K)
        for u, d in enumerate(datas):
            assert np.array_equal(out[u], probs[:d.shape[1], u, :].T)


# ------------------------------------------------------------------------------------------------ accumulation
def _small(maxUtts, reg=0.0, uni=False, k=2, dropout=0.0):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20, numTemporal=k,
                           unidirectional=uni, cell="lstm", dropout=dropout)
    nn.initParams()
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
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    print(json.dumps({"lstm_accum_%s" % ("uni" if uni else "bi"): dict(micro=e_micro, shards=e_shard,
                                                                        cost=float(np.max(np.abs(c2 - c1))))}))
    assert np.allclose(c1, c2, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5
    assert g2[-4] == g3[-4] == g1[-4] == 8 and g1[-1] == g2[-1] == g3[-1] == 0


def _train(useGraphs, optimizer="nesterov", dropout=0.0, steps=5, uni=False):
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
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False, optimizer=optimizer)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn.params.cpu().numpy(), np.array(opt.costt), opt


@pytest.mark.parametrize("optimizer,dropout,uni", [("nesterov", 0.0, False), ("adam", 0.0, True),
                                                   ("nesterov", 0.3, False)])
def test_graph_replay_is_bit_identical_to_eager_steps(optimizer, dropout, uni, cuda):
    """Graph replay against eager steps, also with Adam and with dropout on the ReLU layers of the LSTM net."""
    p_g, c_g, opt_g = _train(True, optimizer, dropout, uni=uni)
    p_e, c_e, opt_e = _train(False, optimizer, dropout, uni=uni)
    print(json.dumps({"lstm_graph_%s_p%g_%s" % (optimizer, dropout, "uni" if uni else "bi"):
                      dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1 and len(opt_e._graphs) == 0
    assert np.array_equal(p_g, p_e) and np.array_equal(c_g, c_e)
    assert np.isfinite(p_g).all()


def test_adam_trains_an_lstm_net(cuda):
    """Twenty Adam steps on one minibatch lower its cost."""
    _, costs, _ = _train(True, "adam", steps=20)
    print(json.dumps({"lstm_adam_costs": costs.tolist()}))
    assert np.isfinite(costs).all() and costs[-1] < 0.9 * costs[0]


def test_dropout_masks_only_the_relu_layers_of_an_lstm_net(cuda):
    """With p = 0.5: the ReLU hidden layers of a training call are dropped (and rescaled), the gradient equals the oracle's back-propagation through the GPU's own (dropped) activations with the
    delta of each dropped layer scaled by 1/(1-p), and the forward-only probabilities are those of the net without
    dropout."""
    import torch
    p = 0.5
    datas, labelss = _ragged()
    nn = _small(8, 0.0, False, k=1, dropout=p)
    ref = _small(8, 0.0, False, k=1)
    nn.costAndGradBatch(datas, labelss)
    ref.costAndGradBatch(datas, labelss)
    B, Tmax = 8, 60
    lens = [d.shape[1] for d in datas]
    acts = workspace_activations(nn, B, Tmax)
    ref_acts = workspace_activations(ref, B, Tmax)
    X = {i: acts[0, i] for i in range(1, 6)}
    Xr = {i: ref_acts[0, i] for i in (1, 3, 4)}
    kept = X[1] != 0        # layer 1 sees the same input in both nets: its kept units are the undropped ones times 2
    assert np.array_equal(X[1][kept], Xr[1][kept] * np.float32(2.0))
    for i in (1, 3, 4):     # about half of each ReLU layer's non-zero units are dropped
        frac = (X[i] != 0).sum() / (Xr[i] != 0).sum()
        assert 0.35 < frac < 0.65, (i, frac)
    # the oracle through the GPU's activations, the dropped layers' deltas scaled by 1/(1-p)
    on = Net(13, 11, 64, 4, 60, temporalLayer=2, cell="lstm", dropout=p)
    on.stack = [[w.cpu().numpy().astype(np.float64), b.cpu().numpy().astype(np.float64)] for w, b in nn.stack]
    tot = [[np.zeros_like(w), np.zeros_like(b)] for w, b in on.stack]
    for u in range(B):
        a = lambda what, i: acts[what, i][:lens[u], u].T        # noqa: E731
        hs = [a(1, 2), a(2, 2)]
        g_acts = [a(0, i) for i in range(1, 6)]
        g_acts[1] = hs[0].astype(np.float64) + hs[1]
        _, g, _ = on.costAndGradGiven(datas[u], labelss[u], g_acts, [(a(0, 2), [a(4, 2), a(5, 2)], hs)])
        for (a_, b), (x, y) in zip(tot, g):
            a_ += x
            b += y
    errs = [_rel(dw.cpu().numpy().reshape(a.shape), a) for (dw, _), (a, _) in zip(nn.grad, tot) if np.any(a)]
    inf_nn = _small(8, 0.0, False, k=1, dropout=p)
    pr = [x.copy() for x in inf_nn.forwardBatch(datas)]
    pr0 = ref.forwardBatch(datas)
    print(json.dumps({"lstm_dropout": dict(grad_given_frob_max=max(errs))}))
    assert max(errs) <= GRAD_TOL, errs
    assert all(np.array_equal(a, b) for a, b in zip(pr, pr0))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests_an_lstm_net(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--cell", "lstm", "--epochs", "1",
            "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16", "--rawDim", "20",
            "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1",
            "--runDir", str(tmp_path / "runs"), "--quiet"]
    _, net = runNNet.run(args)
    assert net.cell == "lstm" and tuple(net.stack[4][0].shape) == (256, 64) and tuple(net.stack[1][0].shape) == (512, 64)
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["cell"] == "lstm"
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.cell == "lstm" and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert tnet.cell == "lstm" and not tnet.train
    assert np.array_equal(tnet.params.cpu().numpy(), p_epoch0)
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16
    # a relu net cannot load the LSTM checkpoint
    import nnets.brnnet as brnnet
    relu = brnnet.NNet(16, 9, 64, 3, 40, temporalLayer=2, train=False)
    relu.initParams()
    import pickle
    with open(os.path.join(run_dir, "params.pk"), "rb") as fid:
        pickle.load(fid)
        with pytest.raises(ValueError, match="cell"):
            relu.fromFile(fid)


def test_a_width_the_device_cannot_hold_is_refused(cuda):
    import _ctcb
    from _ctcb import lib
    cfg = _ctcb.BrnnConfig(41, 32, 2048, 3, 2, 50, 8, 10, 0.0, 20.0, 0, 1, 1)
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    msg = lib.ctcb_last_error().decode()
    print(json.dumps({"lstm_refused": msg}))
    assert "layerSize 2048" in msg and "co-resident" in msg
    with pytest.raises(ValueError, match="2048"):
        import nnets.brnnet as brnnet
        brnnet.NNet(41, 32, 2048, 3, 50, temporalLayer=2, cell="lstm")
