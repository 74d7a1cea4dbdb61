"""GPU tests of stacked temporal layers (numTemporal = k > 1) on one H100.

Parity against the float64 restatement (tests/net_oracle.py, compared by tests/net_check.py) with the criteria of
test_configs_gpu.py: per-utterance cost <= 1e-4; every activation array, For_j / Back_j of each temporal layer included
(read back through ctcb_brnn_activation_offset), within 1e-4 of the oracle's relative to its largest magnitude; every
gradient tensor within 1e-4 (Frobenius) of the oracle's back-propagation through the GPU's own activations; the plain
comparison (oracle with its own float64 masks) printed and bounded: 1e-4 where the sweeps run on FFMA, 1e-2 at H = 1024,
where float32 noise flips the ReLU / clip mask of units near a kink (test_configs_gpu.py) and each flip reaches the
layers below through every stacked recurrence (measured 3.2e-3 and 5.4e-3, while the gradients given the GPU's
activations agree to 1.4e-5). The cases cover each sweep family, checked with ctcb_debug_sweep_plan, bi- and
uni-directional layers, k = 2 and 3, a ragged batch, T = 1 and a block that ends at the top hidden layer. Then: the bits
of k = 1 against a config without the field, forward-only against training probabilities, micro-batches, shards with L2,
CUDA-graph replay, two ranks over NCCL, and runNNet end to end. Each comparison prints its measured errors as one JSON
line (pytest -s)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COST_TOL, FWD_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-4

# sweep: the plan family each case must run (ctcb_debug_sweep_plan kernel: 0 generic, 1 cluster, 2 tensor-core)
CASES = {
    "cluster_h256_bi_k2": dict(H=256, N=4, tl=1, k=2, T=60, B=6, L=12, sweep=1),
    "cluster_h256_uni_k3_ragged": dict(H=256, N=4, tl=1, k=3, T=50, B=7, L=10, uni=True, ragged=True, sweep=1),
    "generic_h96_bi_k3_ragged": dict(H=96, N=4, tl=1, k=3, T=45, B=5, L=9, ragged=True, sweep=0),
    "generic_h96_uni_k2": dict(H=96, N=3, tl=1, k=2, T=30, B=4, L=8, uni=True, sweep=0),
    "tc_h1024_bi_k2_ragged": dict(H=1024, N=4, tl=2, k=2, T=64, B=8, L=12, ragged=True, sweep=2),
    "tc_h1024_uni_k3": dict(H=1024, N=4, tl=1, k=3, T=40, B=8, L=8, uni=True, sweep=2),
    "cluster_h256_bi_k3_T1": dict(H=256, N=4, tl=1, k=3, T=1, B=4, L=1, sweep=1),
    "cluster_h256_bi_k2_top_block": dict(H=256, N=3, tl=2, k=2, T=40, B=4, L=8, top=True, sweep=1),
}
D, K = 41, 32


def _kwargs(c):
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make case c."""
    return dict(temporalLayer=c["tl"], numTemporal=c["k"], unidirectional=bool(c.get("uni")),
                allowTopTemporal=bool(c.get("top")))


def _batch(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    if c.get("ragged"):
        rng = np.random.RandomState(seed)
        lens = [int(x) for x in rng.randint(int(0.6 * T), T + 1, size=B)]
        lens[0] = T
        nlabs = [int(x) for x in rng.randint(max(1, L // 3), L + 1, size=B)]
    else:
        lens, nlabs = [T] * B, [L] * B
    return lens, recipes.synth_batch(D, K, lens, nlabs, seed=33)


@pytest.mark.parametrize("name", list(CASES))
def test_stacked_net_matches_float64_oracle(name, cuda):
    import nnets.brnnet as brnnet
    from _ctcb import lib, check
    c = CASES[name]
    H, N, tl, k, B = c["H"], c["N"], c["tl"], c["k"], c["B"]
    uni = bool(c.get("uni"))
    plan = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_sweep_plan(H, B, 1 if uni else 2, plan))
    assert plan[0] == c["sweep"], (list(plan), c["sweep"])
    lens, (datas, labelss) = _batch(c)
    Tmax = max(lens)
    np.random.seed(33)
    on = Net(D, K, H, N, c["T"], **_kwargs(c))
    on.initParams()
    np.random.seed(33)
    nn = brnnet.NNet(D, K, H, N, c["T"], maxUtts=B, maxLabels=c["L"], **_kwargs(c))
    nn.initParams()
    assert nn.numTemporal == k and len(nn.stack) == len(on.stack)
    for (w, _), (ow, _) in zip(nn.stack, on.stack):         # same draws, same order
        assert np.array_equal(w.cpu().numpy(), ow.astype(np.float32))
    batch = nn._batch.pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, want_probs=True)
    probs_train = nn._probs_view(B, Tmax).clone()
    assert nn.stats.cpu().numpy()[3] == 0
    r = compare(nn, on, datas, labelss, lens)
    if c["T"] == 1:     # one frame: no recurrence, the recurrent gradients are exactly zero on both sides
        assert all(np.abs(dw.cpu().numpy()).max() == 0 for dw, _ in nn.grad[N + 1:])
    # forward-only probabilities of the same net are the training call's, bit for bit
    probs_fwd = nn._forward_device(batch)
    same_probs = bool(np.array_equal(_bits(probs_fwd), _bits(probs_train)))

    assert not r["skips_own"].any()
    cost_err = r["cost_own"]
    fwd_err = max(r["fwd"]["X"] + [r["fwd"]["For"], r["fwd"].get("Back", 0.0)])
    tensors = [t for t in range(len(r["grad_given"])) if t % 2 == 0 or t // 2 <= N]    # matrices, the maps' biases
    given = [r["grad_given"][t] for t in tensors]
    plain = [r["grad_plain"][t] for t in tensors]
    print(json.dumps({name: dict(config=c, cost_rel_err_max=cost_err, forward_activation_rel_err_max=fwd_err,
                                 grad_rel_err_given_gpu_activations_max=max(given),
                                 grad_rel_err_vs_float64_masks_max=max(plain), grad_rel_err_vs_float64_masks=plain,
                                 forward_only_probs_bit_identical=same_probs)}))
    assert same_probs
    assert cost_err <= COST_TOL, cost_err
    assert fwd_err <= FWD_TOL, fwd_err
    assert max(given) <= GRAD_TOL, given
    assert max(plain) <= (1e-2 if H >= 1024 else 1e-4), plain


def test_one_temporal_layer_gives_the_bits_of_a_config_without_the_field(cuda):
    """numTemporal = 1 (what NNet passes) against a handle made from the 11-member initialiser (numTemporal = 0):
    probabilities, costs, gradient and statistics tail, bit for bit, on a ragged batch with L2."""
    import _ctcb
    import nnets.brnnet as brnnet
    from _ctcb import lib, check
    c = dict(H=256, N=3, tl=2, k=1, T=50, B=6, L=10, ragged=True)
    lens, (datas, labelss) = _batch(c)
    np.random.seed(4)
    nn = brnnet.NNet(D, K, c["H"], c["N"], c["T"], maxUtts=c["B"], maxLabels=c["L"], reg=1e-2, **_kwargs(c))
    nn.initParams()
    batch = nn._batch.pack(datas, labelss).upload()
    snaps = []
    for cfg in (nn._cfg, _ctcb.BrnnConfig(D, K, 256, 3, 2, 50, 6, 10, 1e-2, 20.0, 0)):
        assert cfg.numTemporal in (0, 1)
        h = ctypes.c_void_p()
        check(lib.ctcb_brnn_create(ctypes.byref(cfg), ctypes.byref(h)))
        own, nn._h = nn._h, h
        try:
            nn.costAndGradDevice(batch, want_probs=True)
            cuda.cuda.synchronize()
            snaps.append((_bits(nn._probs_view(batch.B, batch.Tmax)), _bits(nn.grads_ext[:nn.nparams + 6]),
                          _bits(nn._out[:batch.B])))
        finally:
            nn._h = own
            lib.ctcb_brnn_destroy(h)
    assert snaps[0][1].size == snaps[1][1].size
    for a, b in zip(*snaps):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ accumulation
def _small_net(kind, maxUtts, k, reg=0.0, N=4, tl=1, H=64):
    import nnets.brnnet
    import nnets.rnnet
    np.random.seed(4)
    if kind == "uni":
        nn = nnets.rnnet.NNet(13, 11, H, N, 60, temporalLayer=tl, maxUtts=maxUtts, maxLabels=20, numTemporal=k)
    else:
        nn = nnets.brnnet.NNet(13, 11, H, N, 60, temporalLayer=tl, reg=reg, maxUtts=maxUtts, maxLabels=20,
                               numTemporal=k)
    nn.initParams()
    return nn


def _ragged(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


def _grads(nn):
    return [(dw.cpu().numpy().astype(np.float64), db.cpu().numpy().astype(np.float64)) for dw, db in nn.grad]


@pytest.mark.parametrize("kind,k,reg", [("bi", 3, 1e-2), ("uni", 2, 0.0), ("uni", 3, 0.0)])
def test_two_micro_batches_match_one_call(kind, k, reg, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    datas, labelss = _ragged()
    full = _small_net(kind, 8, k, reg)
    c1, _, s1 = full.costAndGradBatch(datas, labelss)
    g1, t1 = _grads(full), full.stats.cpu().numpy().astype(np.float64)
    split = _small_net(kind, 4, k, reg)
    c2, _, s2 = split.costAndGradBatch(datas, labelss)
    g2, t2 = _grads(split), split.stats.cpu().numpy().astype(np.float64)
    errs = [e for (a, b), (x, y) in zip(g2, g1) for e in (_rel(a, x), _rel(b, y))]
    cost_err = float(np.max(np.abs(c2 - c1) / np.abs(c1)))
    # the FIRST part alone is a plain call on its micro-batch (reg = 0: no L2 term that only LAST adds)
    nn = _small_net(kind, 4, k, 0.0)
    batch = nn._batch.pack(datas[:4], labelss[:4]).upload()
    nn.costAndGradDevice(batch)
    ref = (_bits(nn.grads_ext[:nn.nparams + 4]), _bits(nn._out[:4]), _bits(nn._out[nn.maxUtts:nn.maxUtts + 4]))
    for w, b in nn.grad:        # NaN into every tensor (the alignment gaps between them are never written)
        w.fill_(float("nan"))
        b.fill_(float("nan"))
    nn.stats.fill_(float("nan"))
    st = _ctcb.current_stream()
    check(lib.ctcb_brnn_cost_and_grad_part(
        nn._h, ptr(batch.d_feats), ptr(batch.d_lens), ptr(batch.d_labels), ptr(batch.d_off), 4, batch.Tmax,
        ptr(nn.params), ptr(nn.grads), ptr(nn._cost[:4]), ptr(nn._skip[:4]), None, None, ptr(nn.stats),
        _ctcb.PART_FIRST, ptr(nn._ws), nn._ws.numel(), st))
    got = (_bits(nn.grads_ext[:nn.nparams + 4]), _bits(nn._out[:4]), _bits(nn._out[nn.maxUtts:nn.maxUtts + 4]))
    first_same = all(np.array_equal(a, b) for a, b in zip(ref, got))
    print(json.dumps({"stack_accum_%s_k%d" % (kind, k): dict(grad_rel_err_max=max(errs), cost_rel_err_max=cost_err,
                                                            first_part_bit_identical=first_same)}))
    assert np.array_equal(s1, s2) and not s1.any()
    assert t2[0] == t1[0] == 8 and t2[3] == t1[3] == 0 and abs(t2[1] - t1[1]) <= 1e-6 * abs(t1[1])
    assert cost_err <= 1e-6
    assert max(errs) <= 1e-5, errs
    assert first_same


def test_two_shards_summed_equal_the_full_batch_with_l2(cuda):
    """Deferred L2 on two shards, summed, reg*W applied once: the full batch's gradient, every recurrent matrix's L2
    counted once.  The bound is the fp32 summation-order bound of the micro-batch comparison (calls of 4 utterances
    against one of 8; measured 2.7e-6), and reg is large enough that the L2 term of each recurrent matrix is over ten
    times that bound, so a missing or doubled one would fail."""
    import _ctcb
    from _ctcb import lib, check, ptr
    import parallel
    reg = 1e-1
    datas, labelss = _ragged()
    full = _small_net("bi", 8, 3, reg)
    full.costAndGradBatch(datas, labelss)
    g_full = full.grads_ext[:full.nparams + 4].clone()
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small_net("bi", 4, 3, reg)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    cuda.cuda.synchronize()
    a, b = total.cpu().numpy().astype(np.float64), g_full.cpu().numpy().astype(np.float64)
    err = _rel(a[:-4], b[:-4])
    # each recurrent matrix alone, where a missing or doubled L2 term would show
    rec, l2 = [], []
    off, r, cc = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    for idx in range(2 * 5, lib.ctcb_brnn_num_tensors(ctypes.byref(full._cfg)), 2):
        check(lib.ctcb_brnn_tensor_info(ctypes.byref(full._cfg), idx, ctypes.byref(off), ctypes.byref(r),
                                        ctypes.byref(cc)))
        sl = slice(off.value, off.value + r.value * cc.value)
        rec.append(_rel(a[sl], b[sl]))
        w = full.params.cpu().numpy().astype(np.float64)[sl]
        l2.append(float(np.linalg.norm(reg * w) / np.linalg.norm(b[sl])))
    print(json.dumps({"stack_two_shards_l2": dict(grad_rel_err=err, recurrent_rel_err=rec, recurrent_l2_share=l2)}))
    assert len(rec) == 6
    assert err < 1e-5 and max(rec) < 1e-5
    # a recurrent matrix whose L2 term were missing or doubled would be off by far more than the bound above
    assert min(l2) > 10 * 1e-5
    assert a[-4] == b[-4] == 8 and abs(a[-3] - b[-3]) / abs(b[-3]) < 1e-6 and a[-1] == b[-1] == 0


def _train(useGraphs, steps=6, k=3, kind="bi"):
    import random
    import sgd
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small_net(kind, 8, k, 1e-2 if kind == "bi" else 0.0)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    import torch
    torch.cuda.synchronize()
    return nn.params.cpu().numpy(), opt._vflat.cpu().numpy(), np.array(opt.costt), opt


@pytest.mark.parametrize("kind,k", [("bi", 3), ("uni", 3)])
def test_graph_replay_of_stacked_steps_is_bit_identical(kind, k, cuda):
    p_g, v_g, c_g, opt_g = _train(True, k=k, kind=kind)
    p_e, v_e, c_e, opt_e = _train(False, k=k, kind=kind)
    print(json.dumps({"stack_graph_%s_k%d" % (kind, k): dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1 and len(opt_e._graphs) == 0
    assert np.array_equal(p_g, p_e) and np.array_equal(v_g, v_e) and np.array_equal(c_g, c_e)
    assert np.isfinite(p_g).all()


# ------------------------------------------------------------------------------------------------ two ranks
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
lens = [25, 30, 18, 30, 22, 27, 16, 29]
datas, labelss = recipes.synth_batch(13, 11, lens, [6, 8, 4, 9, 5, 7, 3, 8], seed=9)
keys = ["k%%d" %% i for i in range(len(lens))]
dd = dict(zip(keys, datas)); alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
np.random.seed(2); random.seed(33)
nn = rnnet.NNet(13, 11, 64, 4, 30, temporalLayer=1, reg=1e-3, maxUtts=parallel.per_rank_capacity(7, world),
                maxLabels=10, numTemporal=3)
nn.initParams()
opt = sgd.SGD(nn, 30, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=7, verbose=False)
for _ in range(2):
    opt.run(dd, alis, list(keys), None)     # steps of 7 and 1 utterances: the second leaves one rank's shard empty
torch.cuda.synchronize()
np.save(os.path.join(sys.argv[1], "params_w%%d_r%%d.npy" %% (world, rank)), nn.params.cpu().numpy())
if world > 1:
    dist.barrier(); dist.destroy_process_group()
'''


def test_two_rank_stacked_steps_match_single_gpu(cuda, tmp_path):
    if cuda.cuda.device_count() < 2:
        pytest.skip("two-rank NCCL test of a stacked net: needs 2 GPUs, %d visible" % cuda.cuda.device_count())
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", "29627", str(script), str(tmp_path)],
                           env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        _, e1 = p1_.communicate(timeout=600)
        _, e2 = p2_.communicate(timeout=600)
    finally:
        for p_ in (p1_, p2_):
            if p_.poll() is None:
                p_.kill()
    assert p1_.returncode == 0, e1[-2000:]
    assert p2_.returncode == 0, e2[-2000:]
    p1 = np.load(tmp_path / "params_w1_r0.npy")
    p20, p21 = np.load(tmp_path / "params_w2_r0.npy"), np.load(tmp_path / "params_w2_r1.npy")
    err = float(np.linalg.norm(p20 - p1) / np.linalg.norm(p1))
    print(json.dumps({"stack_dp2": dict(params_rel_err=err)}))
    assert np.array_equal(p20, p21)
    assert err < 1e-5


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests_a_stacked_net(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "64", "--numLayers", "4", "--temporalLayer", "1", "--numTemporal", "2", "--epochs", "1",
            "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16", "--rawDim", "20",
            "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1",
            "--runDir", str(tmp_path / "runs"), "--quiet"]
    _, net = runNNet.run(args)
    assert net.numTemporal == 2 and len(net.stack) == 5 + 4
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["numTemporal"] == 2
    p_epoch0 = net.params.cpu().numpy().copy()
    np.random.seed(33)
    fresh = Net(16, 9, 64, 4, 40, temporalLayer=1, numTemporal=2)
    fresh.initParams()
    assert not np.array_equal(net.stack[5][0].cpu().numpy(), fresh.stack[5][0].astype(np.float32))    # it trained
    cfg["epochs"] = 2                                   # resume: one more epoch
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.numTemporal == 2
    # the stacked model and its optimiser state came back from params.pk (epoch 0 recorded both files as done, so
    # the resumed epoch has nothing left to train)
    p_epoch1 = net2.params.cpu().numpy()
    assert np.array_equal(p_epoch0, p_epoch1)
    assert os.path.exists(os.path.join(run_dir, "params.pk.epoch01"))
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert tnet.numTemporal == 2 and not tnet.train
    assert np.array_equal(tnet.params.cpu().numpy(), p_epoch1)      # the model the resumed run saved
    for fn in (1, 2):
        size = os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn))
        assert size > 9 * 16
    loader = dl.DataLoader(data, 20, 16, data)
    data_dict, _, keys, _ = loader.loadDataFileDict(1)
    probs = tnet.forwardBatch([data_dict[k] for k in keys])
    import pickle
    with open(os.path.join(out, "loglikelihoods_1.pk"), "rb") as f:
        lik = pickle.load(f)
    for k, p in zip(keys, probs):
        with np.errstate(divide="ignore"):
            assert np.array_equal(lik[k], np.log(p))
