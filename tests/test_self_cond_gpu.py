"""GPU tests of self-conditioned CTC (ctcb_brnn_config.selfCondition) on one H100.

The row-softmax backward kernel against float64; the InterCTC test's nine whole nets with random non-zero W_c, b_c
against tests/net_oracle.Net; at W_c = b_c = 0 the InterCTC net; forward-only probabilities bit for bit
with a training call's; micro-batches and emulated shards, forced stalls and graph replay for m below, at and above
the lowest temporal layer; two ranks over NCCL (skipped with fewer than 2 GPUs); checkpoints, check_grad and runNNet.
Each comparison prints its measured numbers as one JSON line (pytest -s)."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from recipes import knobs  # noqa: F401  (fixture)
from net_oracle import Net
from test_inter_ctc_gpu import NETS, D, K, LAM, _batch, _kwargs, _ragged

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("Kc", [1, 31, 32, 33, 62, 128])
@pytest.mark.parametrize("with_add", [False, True])
def test_softmax_backward_kernel_against_float64(Kc, with_add, cuda):
    """out = p (dp - sum p dp) + add, element-wise within (4 + 2K) 2^-24 (p_j (|dp_j| + sum_k p_k |dp_k|) + |add_j|)
    of float64 on the float32 inputs; out aliasing dp gives the same bytes."""
    import _ctcb
    import torch
    from _ctcb import lib, check, ptr
    R = 1000
    rng = np.random.RandomState(Kc + 7 * with_add)
    x = rng.uniform(-30, 30, (R, Kc))
    p = np.exp(x - x.max(axis=1, keepdims=True))
    p = (p / p.sum(axis=1, keepdims=True)).astype(np.float32)
    dp = (rng.standard_normal((R, Kc)) * np.exp(rng.uniform(-3, 3, (R, 1)))).astype(np.float32)
    add = rng.standard_normal((R, Kc)).astype(np.float32) if with_add else None
    P64, D64 = p.astype(np.float64), dp.astype(np.float64)
    ref = P64 * (D64 - (P64 * D64).sum(axis=1, keepdims=True)) + (0.0 if add is None else add.astype(np.float64))
    mag = P64 * (np.abs(D64) + (P64 * np.abs(D64)).sum(axis=1, keepdims=True))
    bound = (4 + 2 * Kc) * 2.0 ** -24 * (mag + (0.0 if add is None else np.abs(add))) + 1e-45
    dev = lambda a: torch.from_numpy(a).cuda()     # noqa: E731
    tp, tdp = dev(p), dev(dp)
    tadd = dev(add) if add is not None else None
    out = torch.empty_like(tp)
    check(lib.ctcb_softmax_rows_backward_f32(ptr(tp), ptr(tdp), ptr(tadd), ptr(out), R, Kc, _ctcb.current_stream()))
    check(lib.ctcb_softmax_rows_backward_f32(ptr(tp), ptr(tdp), ptr(tadd), ptr(tdp), R, Kc, _ctcb.current_stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    ratio = float(np.max(np.abs(got - ref) / bound))
    print(json.dumps({"self_cond_softmax_bwd_K%d_%s" % (Kc, "add" if with_add else "noadd"): dict(err_over_bound=ratio)}))
    assert ratio <= 1.0
    assert np.array_equal(got.view(np.uint32), tdp.cpu().numpy().view(np.uint32))


# ------------------------------------------------------------------------------------------------- whole nets
def _gpu_net(c, B, reg=0.0, cond=True, train=True, lam=LAM):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, selfCondition=cond,
                       **_kwargs(c, reg, lam))


def _set_cond(nn, on=None, seed=8, scale=0.3):
    """Random non-zero W_c and b_c on the device net (and the oracle)."""
    import torch
    rng = np.random.RandomState(seed)
    H = nn.layerSize
    wc = rng.uniform(-scale, scale, (H, nn.outputDim)).astype(np.float32)
    bc = rng.uniform(-0.1, 0.1, (H, 1)).astype(np.float32)
    nn.stack[-1][0].copy_(torch.from_numpy(wc))
    nn.stack[-1][1].copy_(torch.from_numpy(bc))
    if on is not None:
        on.stack[-1][0][...] = wc
        on.stack[-1][1][...] = bc


def _pair(c, B, reg, wc=True):
    """The device net and its oracle with the same parameters (random peephole weights, W_c and b_c)."""
    import torch
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = Net(D, K, c["H"], c["N"], c["T"], selfCondition=True, **_kwargs(c, reg))
    on.initParams()
    if c.get("peep"):
        n = nn.peepholeEntries()
        rng = np.random.RandomState(8)
        for (w, _), (ow, _) in zip(nn.stack[len(nn.stack) - 1 - n:-1], on.stack[len(on.stack) - 1 - n:-1]):
            x = rng.uniform(-0.5, 0.5, tuple(w.shape)).astype(np.float32)
            w.copy_(torch.from_numpy(x))
            ow[...] = x
    if wc:
        _set_cond(nn, on)
    if nn.dropoutStep is not None:
        nn.dropoutStep.fill_(3)
    on.dropoutStep = 3
    return nn, on


@pytest.mark.parametrize("name", list(NETS))
def test_net_matches_float64_oracle(name, cuda):
    """The device's training call against the float64 net: the main costs, the intermediate nll of every utterance, and
    every gradient tensor (W_c and b_c included) against the back-propagation through the device's own activations,
    X'_m and P."""
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
    print(json.dumps({"self_cond_net_" + name: dict(cost=r["cost_own"], inter_cost=inter,
                                                    grad_given_frob_max=max(grad_err),
                                                    grad_given_elem_max=max(r["grad_given_elem"]),
                                                    grad_cond=grad_err[-2:], grad_plain_max=max(r["grad_plain"]))}))
    assert r["cost_own"] <= 1e-4
    assert inter <= 1e-4
    assert max(grad_err) <= 1e-4, grad_err
    assert np.any(nn.grad[-1][0].cpu().numpy()) and np.any(nn.grad[-1][1].cpu().numpy())


@pytest.mark.parametrize("name", list(NETS))
def test_zero_conditioning_is_the_interctc_net(name, cuda):
    """At W_c = b_c = 0: the costs, the intermediate nll and the probabilities are those of the net without
    conditioning, and every other gradient tensor agrees to 1e-5."""
    import torch
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    np.random.seed(21)
    nn = _gpu_net(c, c["B"])
    nn.initParams()
    np.random.seed(21)
    ref = _gpu_net(c, c["B"], cond=False)
    ref.initParams()
    assert torch.equal(nn.params[:ref.nparams], ref.params) and not torch.any(nn.params[ref.nparams:])
    for net in (nn, ref):
        if net.dropoutStep is not None:
            net.dropoutStep.fill_(3)
    c1, _, s1 = nn.costAndGradBatch(datas, labelss)
    c0, _, s0 = ref.costAndGradBatch(datas, labelss)
    assert np.array_equal(c1, c0) and np.array_equal(s1, s0)
    assert np.array_equal(nn.interCosts, ref.interCosts) and np.array_equal(nn.interSkips, ref.interSkips)
    errs = [_rel(x.cpu().numpy(), y.cpu().numpy()) for a, b in zip(nn.grad[:-1], ref.grad) for x, y in zip(a, b)]
    print(json.dumps({"self_cond_zero_" + name: dict(grad_rel_max=max(errs))}))
    assert max(errs) <= 1e-5, errs
    pa, pb = nn.forwardBatch(datas), ref.forwardBatch(datas)
    assert all(np.array_equal(x, y) for x, y in zip(pa, pb))


@pytest.mark.parametrize("name", [n for n in NETS if not NETS[n].get("p")])
def test_forward_only_probabilities_are_the_training_calls(name, cuda):
    """A forward-only call conditions in place what a training call conditions in a copy, with the same launches and
    plans: the probabilities are the same bytes."""
    import torch
    c = NETS[name]
    lens, (datas, labelss) = _batch(c)
    nn, _ = _pair(c, c["B"], 0.0)
    batch = nn._batch.pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, want_probs=True)
    pt = nn._probs_view(batch.B, nn.frames(batch.Tmax)).clone()
    pf = nn._forward_device(batch).clone()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(pt), _bits(pf))
    # and the conditioning changes them: W_c = 0 gives other probabilities
    nn.stack[-1][0].zero_()
    p0 = nn._forward_device(batch).clone()
    assert not np.array_equal(_bits(p0), _bits(pf))


# ------------------------------------------------------------------------------------------- step consistency
def _small(maxUtts, m=1, uni=False, cell="lstm", cond=True, reg=1e-2):
    """N = 4 with temporal layers 2 and 3: m = 1 lies below the lowest, 2 at it (below the highest), 3 at the highest."""
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20, numTemporal=2,
                           unidirectional=uni, cell=cell, peephole=cell == "lstm", dropout=0.2, interLayer=m,
                           interWeight=LAM, selfCondition=cond)
    nn.initParams()
    if cond:
        _set_cond(nn, seed=m)
    return nn


CASES = [dict(uni=False, m=1, cell="lstm"), dict(uni=True, m=2, cell="relu"), dict(uni=True, m=3, cell="lstm"),
         dict(uni=False, m=2, cell="relu")]


@pytest.mark.parametrize("case", CASES)
def test_micro_batches_and_two_shards_match_one_call(case, cuda):
    """Three micro-batches and two emulated shards against one call: the gradient, the statistics tail and the
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
    wc = slice((full.stack[-1][0].data_ptr() - full.params.data_ptr()) // 4, full.nparams)     # W_c and b_c
    e_cond = max(_rel(g2[wc], g1[wc]), _rel(g3[wc], g1[wc]))
    print(json.dumps({"self_cond_accum_%s_m%d_%s" % ("uni" if case["uni"] else "bi", case["m"], case["cell"]):
                      dict(micro=e_micro, shards=e_shard, cond_tensors=e_cond)}))
    assert np.any(g1[wc])
    assert np.allclose(c1, c2, rtol=1e-6) and np.allclose(i1, split.interCosts, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5 and e_cond < 1e-5
    for g in (g2, g3):
        assert np.array_equal(g[-6:][[0, 2, 3, 5]], g1[-6:][[0, 2, 3, 5]])
        assert np.allclose(g[-6:][[1, 4]], g1[-6:][[1, 4]], rtol=1e-5)


@pytest.mark.parametrize("mode", ["main", "side"])
@pytest.mark.parametrize("case", CASES)
def test_forced_stalls_keep_every_byte(mode, case, knobs, cuda):
    datas, labelss = _ragged()
    want = _small(8, **case)
    want.dropoutStep.fill_(2)
    cw, _, _ = want.costAndGradBatch(datas, labelss)
    gw, iw = _bits(want.grads_ext), want.interCosts.copy()
    knobs("CTCB_STALL", mode)
    knobs("CTCB_STALL_US", "500")
    got = _small(8, **case)
    got.dropoutStep.fill_(2)
    cg, _, _ = got.costAndGradBatch(datas, labelss)
    assert np.array_equal(cw, cg) and np.array_equal(gw, _bits(got.grads_ext)) and np.array_equal(iw, got.interCosts)


def _train(useGraphs, m, steps=6):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8, m=m, reg=1e-3)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn, np.array(opt.costt), opt


@pytest.mark.parametrize("m", [1, 3])
def test_graph_replay_is_bit_identical_to_eager_steps(m, cuda):
    nn_g, c_g, opt_g = _train(True, m)
    nn_e, c_e, _ = _train(False, m)
    print(json.dumps({"self_cond_graph_m%d" % m: dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1
    assert np.array_equal(nn_g.params.cpu().numpy(), nn_e.params.cpu().numpy()) and np.array_equal(c_g, c_e)


# ---------------------------------------------------------------------------------------------- two ranks
WORKER = r'''
import os, sys
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tests")]
import numpy as np, torch, torch.distributed as dist
rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
if world > 1:
    dist.init_process_group("nccl")
import random, recipes, nnets.brnnet as rnnet, sgd, parallel
m = int(sys.argv[2])
datas, labelss = recipes.synth_batch(13, 11, [25, 30, 18, 30, 22, 27], [6, 8, 4, 9, 5, 7], seed=9)
keys = ["k%%d" %% i for i in range(6)]
dd = dict(zip(keys, datas)); alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
np.random.seed(2); random.seed(33)
nn = rnnet.NNet(13, 11, 64, 4, 30, temporalLayer=2, numTemporal=2, reg=1e-3,
                maxUtts=parallel.per_rank_capacity(6, world), maxLabels=10, interLayer=m, interWeight=0.5,
                selfCondition=True)
nn.initParams()
opt = sgd.SGD(nn, 30, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=6, verbose=False)
for _ in range(3):
    opt.run(dd, alis, list(keys), None)
torch.cuda.synchronize()
np.save(os.path.join(sys.argv[1], "params_m%%d_w%%d_r%%d.npy" %% (m, world, rank)), nn.params.cpu().numpy())
if world > 1:
    dist.barrier(); dist.destroy_process_group()
'''


@pytest.mark.parametrize("m", [1, 3])
def test_two_rank_step_matches_single_gpu(m, cuda, tmp_path):
    """m = 1 below the lowest temporal layer (the whole gradient exchanged at the end) and m = 3 at the highest (the
    early exchange carries dA's share of W_{N+1}): two ranks over NCCL against one GPU."""
    if cuda.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path), str(m)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", str(29631 + m), str(script), str(tmp_path),
                            str(m)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        _, e1 = p1_.communicate(timeout=600)
        _, e2 = p2_.communicate(timeout=600)
    finally:
        for p_ in (p1_, p2_):
            if p_.poll() is None:
                p_.kill()
    assert p1_.returncode == 0, e1[-2000:]
    assert p2_.returncode == 0, e2[-2000:]
    p1 = np.load(tmp_path / ("params_m%d_w1_r0.npy" % m))
    p20, p21 = np.load(tmp_path / ("params_m%d_w2_r0.npy" % m)), np.load(tmp_path / ("params_m%d_w2_r1.npy" % m))
    assert np.array_equal(p20, p21)
    assert np.linalg.norm(p20 - p1) / np.linalg.norm(p1) < 1e-5


# --------------------------------------------------------------------------------------------------- the rest
def test_checkpoints_are_refused_across_settings(cuda, tmp_path):
    with_ = _small(8, m=2)
    without = _small(8, m=2, cond=False)
    for src, dst, name in ((with_, without, "with.pk"), (without, with_, "without.pk")):
        f = str(tmp_path / name)
        with open(f, "wb") as fid:
            src.toFile(fid)
        with open(f, "rb") as fid:
            with pytest.raises(ValueError, match="selfCondition=%s" % dst.selfCondition):
                dst.fromFile(fid)
    f = str(tmp_path / "with.pk")
    other = _small(8, m=2)
    other.params.zero_()
    with open(f, "rb") as fid:
        other.fromFile(fid)
    assert np.array_equal(other.params.cpu().numpy(), with_.params.cpu().numpy())


def test_check_grad(cuda):
    import nnets.brnnet as brnnet
    datas, labelss = recipes.synth_batch(13, 11, [30], [6], seed=2)
    np.random.seed(5)
    nn = brnnet.NNet(13, 11, 16, 3, 30, temporalLayer=2, cell="lstm", maxLabels=6, interLayer=1, interWeight=0.8,
                     selfCondition=True)
    nn.initParams()
    _set_cond(nn, seed=3, scale=0.1)
    cost, _, _ = nn.costAndGrad(datas[0], labelss[0])
    assert np.isclose(cost, nn._cost[0].item() + np.float32(0.8) * nn.interCosts[0], rtol=1e-6)
    out = np.array(nn.check_grad(datas[0], labelss[0], epsilon=1e-2, maxChecks=4, verbose=False))
    err = np.abs(out[:, 0] - out[:, 1]) / np.maximum(np.abs(out[:, 1]), 5e-2)
    print(json.dumps({"self_cond_check_grad": dict(probes=len(out), rel_err_max=float(err.max()))}))
    assert float(err.max()) < 0.1


def test_run_nnet_trains_resumes_and_tests(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--interLayer", "1", "--interWeight",
            "0.4", "--selfCondition", "--epochs", "1", "--step", "1e-3", "--dataDir", data, "--numFiles", "2",
            "--inputDim", "16", "--rawDim", "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6",
            "--batchSize", "4", "--save_every", "1", "--runDir", str(tmp_path / "runs"), "--quiet"]
    opt, net = runNNet.run(args)
    assert net.selfCondition and opt.costt and np.any(net.stack[-1][0].cpu().numpy())
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["selfCondition"] is True
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.selfCondition and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    arks = {}
    for tag, zero in (("cond", False), ("zero", True)):
        c = load_config(cfg_file)
        if zero:     # the same checkpoint with W_c = b_c = 0: the net without conditioning
            with open(c["in_file"], "rb") as fid:
                state, stack = pickle.load(fid), pickle.load(fid)
            stack[-1] = [np.zeros_like(stack[-1][0]), np.zeros_like(stack[-1][1])]
            c["in_file"] = str(tmp_path / "zero.bin")
            with open(c["in_file"], "wb") as fid:
                pickle.dump(state, fid)
                pickle.dump(stack, fid)
            f = str(tmp_path / "zero_cfg.json")
            dump_config(c, f)
        else:
            f = cfg_file
        out = str(tmp_path / ("arks_" + tag))
        tnet = runNNet.run(["--cfg_file", f, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                            "--maxUtts", "4"])
        assert not tnet.train and tnet.selfCondition and tnet.interLayer == 1
        arks[tag] = [open(os.path.join(out, "loglikelihoods%d.ark" % fn), "rb").read() for fn in (1, 2)]
        assert all(len(a) > 9 * 16 for a in arks[tag])
    assert all(a != b for a, b in zip(arks["cond"], arks["zero"]))
