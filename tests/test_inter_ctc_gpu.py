"""GPU tests of the intermediate CTC loss (ctcb_brnn_config.interLayer) on one H100.

Whole nets against tests/net_oracle.Net (tests/net_check.py): the per-utterance intermediate nll and every
gradient tensor.  Then the two CTCs skipping on their own, the statistics tail, micro-batches and emulated shards,
graph replay and forced stalls bit for bit, forward-only probabilities bit for bit with the net without the loss,
checkpoints in both directions, check_grad, the SGD log line and runNNet.  Each comparison prints its measured numbers
as one JSON line (pytest -s)."""
import json
import os

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net
from recipes import knobs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

D, K = 23, 17
NETS = {
    "bi_relu_m_temporal": dict(H=64, N=3, tl=2, m=2, T=30, B=6, L=8),
    "uni_relu_m_relu_ragged": dict(H=70, N=3, tl=2, m=1, T=25, B=5, L=6, uni=True, ragged=True),
    "bi_lstm_peep_k2_m_temporal": dict(H=64, N=4, tl=2, nt=2, m=3, T=20, B=7, L=6, ragged=True, cell="lstm",
                                       peep=True),
    "uni_lstm_k2_m_temporal": dict(H=64, N=3, tl=1, nt=2, m=1, T=20, B=5, L=6, ragged=True, cell="lstm", uni=True),
    "bi_relu_ln_drop_at_m": dict(H=64, N=4, tl=3, m=2, T=20, B=5, L=6, ragged=True, ln=True, p=0.3),
    "bi_relu_sub_below_m": dict(H=128, N=3, tl=2, m=1, T=24, B=4, L=4, sub=(2, 3)),
    "bi_lstm_sub_stacked_above_m": dict(H=64, N=3, tl=2, m=1, T=21, B=5, L=4, ragged=True, sub=(3, 2), cell="lstm"),
    "uni_relu_sub_at_m": dict(H=64, N=3, tl=2, m=2, T=24, B=5, L=4, ragged=True, sub=(2, 2), uni=True),
    "dnn": dict(H=96, N=3, tl=-1, m=1, T=30, B=6, L=8, ragged=True),
}
LAM = 0.6


def _kwargs(c, reg=0.0, lam=LAM):
    k, L = c.get("sub", (1, 1))
    return dict(temporalLayer=c["tl"], numTemporal=c.get("nt", 1), reg=reg, unidirectional=bool(c.get("uni")),
                cell=c.get("cell", "relu"), peephole=bool(c.get("peep")), layerNorm=bool(c.get("ln")),
                dropout=c.get("p", 0.0), dropoutSeed=5, subsample=k, subsampleLayer=L,
                interLayer=c["m"] if lam else 0, interWeight=lam)


def _gpu_net(c, B, reg=0.0, lam=LAM, train=True):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg, lam))


def _oracle(c, reg, lam=LAM):
    return Net(D, K, c["H"], c["N"], c["T"], **_kwargs(c, reg, lam))


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


def _pair(c, B, reg):
    """The device net and its oracle with the same parameters (random peephole weights where there are any)."""
    import torch
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = _oracle(c, reg)
    on.initParams()
    if c.get("peep"):
        n = nn.peepholeEntries()
        rng = np.random.RandomState(8)
        for (w, _), (ow, _) in zip(nn.stack[len(nn.stack) - n:], on.stack[len(on.stack) - n:]):
            x = rng.uniform(-0.5, 0.5, tuple(w.shape)).astype(np.float32)
            w.copy_(torch.from_numpy(x))
            ow[...] = x
    if nn.dropoutStep is not None:
        nn.dropoutStep.fill_(3)
    on.dropoutStep = 3
    return nn, on


@pytest.mark.parametrize("name", list(NETS))
def test_net_matches_float64_oracle(name, cuda):
    """The device's training call against the float64 net: the main costs, the intermediate nll of every utterance,
    and every gradient tensor against the back-propagation through the device's own activations."""
    import torch
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    nn, on = _pair(c, c["B"], 1e-3)
    nn.costAndGradBatch(datas, labelss)
    torch.cuda.synchronize()
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    assert np.array_equal(r["inter_skips"], r["inter_skips_own"]) and not r["inter_skips"].any()
    inter = r["inter_cost"]
    grad_err = r["grad_given"]
    print(json.dumps({"inter_ctc_net_" + name: dict(cost=r["cost_own"], inter_cost=inter,
                                                    grad_given_frob_max=max(grad_err),
                                                    grad_given_elem_max=max(r["grad_given_elem"]),
                                                    grad_plain_max=max(r["grad_plain"]))}))
    assert r["cost_own"] <= 1e-4
    assert inter <= 1e-4
    assert max(grad_err) <= 1e-4, grad_err


def _stats(nn):
    return nn.stats.cpu().numpy().astype(np.float64)


def test_main_only_skip_keeps_the_intermediate_gradient(cuda):
    """Below the subsampling point the intermediate CTC has T frames and the main one ceil(T / 2): n equal labels need
    2n - 1 frames, so the main CTC alone skips the utterances with 7 and 5 of them.  Skips, nll, the statistics tail and the gradient
    against the oracle, which sums the intermediate gradient of such an utterance too."""
    import torch
    c = dict(NETS["bi_relu_sub_below_m"], B=4, L=8)
    datas, _ = recipes.synth_batch(D, K, [24, 24, 20, 16], [1] * 4, seed=3)
    labelss = [np.array([1, 2, 3], np.int32), np.array([3] * 7, np.int32), np.array([5, 6], np.int32),
               np.array([4] * 5, np.int32)]
    nn, on = _pair(c, 4, 0.0)
    costs, grad, skips = nn.costAndGradBatch(datas, labelss)
    torch.cuda.synchronize()
    o_costs, o_grad, o_skips = on.costAndGradBatch(datas, labelss)
    assert list(skips) == list(o_skips) == [False, True, False, True]
    assert list(nn.interSkips) == list(on.interSkips) == [False, False, False, False]
    st = _stats(nn)
    ok = ~skips
    assert st[0] == 2 and st[2] == 2 and st[5] == 0
    assert np.isclose(st[1], np.sum(costs[ok]), rtol=1e-6) and np.isclose(st[4], np.sum(nn.interCosts), rtol=1e-6)
    assert float(np.max(np.abs(nn.interCosts - on.interCosts) / on.interCosts)) <= 1e-4
    err = [_rel(g.cpu().numpy(), og) for pair, opair in zip(grad, o_grad) for g, og in zip(pair, opair) if np.any(og)]
    print(json.dumps({"inter_ctc_main_skip": dict(grad_rel_max=max(err))}))
    assert max(err) <= 1e-4


def test_intermediate_only_skip(cuda):
    """The reverse: layer 1 of a DNN made a thousand times larger (and layer 2 as much smaller) gives intermediate
    logits so far apart that every label but the top one has probability 0 in float32 and float64, so the intermediate
    CTC skips every utterance while the main one keeps them; the step then has the main gradient alone."""
    import torch
    c = NETS["dnn"]
    lens, (datas, labelss) = _batch(c)
    nn, on = _pair(c, c["B"], 0.0)
    for net_w, scale in ((0, 1e3), (1, 1e-3)):
        nn.stack[net_w][0].mul_(scale)
        on.stack[net_w][0][...] = nn.stack[net_w][0].cpu().numpy()
    ref = _gpu_net(c, c["B"], lam=0.0)
    ref.initParams()
    ref.params.copy_(nn.params)
    costs, _, skips = nn.costAndGradBatch(datas, labelss)
    torch.cuda.synchronize()
    on.costAndGradBatch(datas, labelss)
    assert not skips.any() and nn.interSkips.all() and on.interSkips.all()
    st = _stats(nn)
    assert st[4] == 0 and st[5] == c["B"]
    rc, _, rs = ref.costAndGradBatch(datas, labelss)
    # the skipped head adds D_aux = 0 with beta = 1: the same values (a -0.0 may become +0.0)
    assert np.array_equal(costs, rc) and np.array_equal(nn.grads.cpu().numpy(), ref.grads.cpu().numpy())


def _small(maxUtts, lam=LAM, uni=False, reg=1e-2, m=1, cell="lstm"):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20, numTemporal=2,
                           unidirectional=uni, cell=cell, peephole=cell == "lstm", dropout=0.2,
                           interLayer=m if lam else 0, interWeight=lam)
    nn.initParams()
    return nn


def _ragged(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


@pytest.mark.parametrize("case", [dict(uni=False, m=1, cell="lstm"), dict(uni=True, m=2, cell="relu"),
                                  dict(uni=True, m=3, cell="lstm")])
def test_micro_batches_and_two_shards_match_one_call(case, cuda):
    """Three micro-batches and two emulated shards against one call: the gradient, the 6-float statistics tail and the
    intermediate nll agree to the reordering of the sums."""
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    datas, labelss = _ragged()
    full = _small(8, **case)
    full.dropoutStep.fill_(4)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    i1 = full.interCosts.copy()
    g1 = full.grads_ext[:full.nparams + 6].cpu().numpy().astype(np.float64)
    split = _small(3, **case)
    split.dropoutStep.fill_(4)
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 6].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4, **case)
        nn.dropoutStep.fill_(4)
        nn.dropoutShard = (rank, 2)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 6].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    e_micro, e_shard = _rel(g2[:-6], g1[:-6]), _rel(g3[:-6], g1[:-6])
    print(json.dumps({"inter_ctc_accum_%s_m%d_%s" % ("uni" if case["uni"] else "bi", case["m"], case["cell"]):
                      dict(micro=e_micro, shards=e_shard)}))
    assert np.allclose(c1, c2, rtol=1e-6) and np.allclose(i1, split.interCosts, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5
    for g in (g2, g3):
        assert np.array_equal(g[-6:][[0, 2, 3, 5]], g1[-6:][[0, 2, 3, 5]])
        assert np.allclose(g[-6:][[1, 4]], g1[-6:][[1, 4]], rtol=1e-5)
    assert np.isclose(g1[-2], np.sum(i1), rtol=1e-5)


def _train(useGraphs, steps=6, verbose=False):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8, reg=1e-3, m=3)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=verbose)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn, np.array(opt.costt), opt


def test_graph_replay_is_bit_identical_to_eager_steps(cuda):
    nn_g, c_g, opt_g = _train(True)
    nn_e, c_e, opt_e = _train(False)
    print(json.dumps({"inter_ctc_graph": dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1
    assert np.array_equal(nn_g.params.cpu().numpy(), nn_e.params.cpu().numpy()) and np.array_equal(c_g, c_e)


def test_log_line_reports_the_intermediate_cost(cuda, capsys):
    nn, costs, opt = _train(False, steps=2, verbose=True)
    out = capsys.readouterr().out.splitlines()
    lines = [l for l in out if l.startswith("Iter ")]
    assert len(lines) == 2 and all(", InterCost=" in l and ", ExpCost=" in l for l in lines), lines
    inter = float(lines[-1].split("InterCost=")[1].split(",")[0])
    assert np.isfinite(inter) and inter > 0
    off = _small(8, lam=0.0)
    assert off.statsFloats == 4 and nn.statsFloats == 6


@pytest.mark.parametrize("mode", ["main", "side"])
def test_forced_stalls_keep_every_byte(mode, knobs, cuda):
    datas, labelss = _ragged()
    want = _small(8, m=3)
    want.dropoutStep.fill_(2)
    cw, _, _ = want.costAndGradBatch(datas, labelss)
    gw, iw = _bits(want.grads_ext), want.interCosts.copy()
    knobs("CTCB_STALL", mode)
    knobs("CTCB_STALL_US", "500")
    got = _small(8, m=3)
    got.dropoutStep.fill_(2)
    cg, _, _ = got.costAndGradBatch(datas, labelss)
    assert np.array_equal(cw, cg) and np.array_equal(gw, _bits(got.grads_ext)) and np.array_equal(iw, got.interCosts)


def test_forward_only_probabilities_are_those_of_the_net_without_the_loss(cuda):
    """Forward-only calls never run the head: the probabilities of a training net with the loss and of forward-only
    nets with and without it are the same bytes."""
    datas, _ = _ragged()
    with_ = _small(8, m=2)
    without = _small(8, lam=0.0)
    without.params.copy_(with_.params)
    a, b = with_.forwardBatch(datas), without.forwardBatch(datas)
    assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


def test_checkpoints_load_in_both_directions(cuda, tmp_path):
    datas, labelss = _ragged()
    with_ = _small(8, m=1)
    without = _small(8, lam=0.0)
    np.random.seed(9)
    without.initParams()
    f = str(tmp_path / "with.pk")
    with open(f, "wb") as fid:
        with_.toFile(fid)
    with open(f, "rb") as fid:
        without.fromFile(fid)
    assert np.array_equal(without.params.cpu().numpy(), with_.params.cpu().numpy())
    np.random.seed(10)
    without.initParams()
    g = str(tmp_path / "without.pk")
    with open(g, "wb") as fid:
        without.toFile(fid)
    with open(g, "rb") as fid:
        with_.fromFile(fid)
    assert np.array_equal(without.params.cpu().numpy(), with_.params.cpu().numpy())
    with_.costAndGradBatch(datas, labelss)
    assert np.isfinite(with_.interCosts).all()


def test_check_grad(cuda):
    import nnets.brnnet as brnnet
    datas, labelss = recipes.synth_batch(13, 11, [30], [6], seed=2)
    np.random.seed(5)
    nn = brnnet.NNet(13, 11, 16, 3, 30, temporalLayer=2, cell="lstm", maxLabels=6, interLayer=1, interWeight=0.8)
    nn.initParams()
    cost, _, _ = nn.costAndGrad(datas[0], labelss[0])
    assert np.isclose(cost, nn._cost[0].item() + np.float32(0.8) * nn.interCosts[0], rtol=1e-6)
    out = np.array(nn.check_grad(datas[0], labelss[0], epsilon=1e-2, maxChecks=4, verbose=False))
    err = np.abs(out[:, 0] - out[:, 1]) / np.maximum(np.abs(out[:, 1]), 5e-2)
    print(json.dumps({"inter_ctc_check_grad": dict(probes=len(out), rel_err_max=float(err.max()))}))
    assert float(err.max()) < 0.1


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--interLayer", "1", "--interWeight",
            "0.4", "--epochs", "1", "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16",
            "--rawDim", "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4",
            "--save_every", "1", "--runDir", str(tmp_path / "runs"), "--quiet"]
    opt, net = runNNet.run(args)
    assert net.interLayer == 1 and net.interWeight == 0.4 and opt.costt
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["interLayer"] == 1 and cfg["interWeight"] == 0.4
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    # the run resumes behind its last checkpoint, with the loss on
    assert net2.interLayer == 1 and net2.interWeight == 0.4
    assert np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert not tnet.train and tnet.interLayer == 0
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16
    assert np.isfinite(net2.params.cpu().numpy()).all()
