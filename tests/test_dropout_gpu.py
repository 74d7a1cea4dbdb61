"""GPU tests of inverted dropout on the ReLU hidden layers (ctcb_brnn_set_dropout, NNet(dropout=p), SGD) on one H100.

  * p = 0 is today's behaviour: a handle given p = 0 (and any utterance map) issues the launches and writes the bits of
    one that never heard of dropout.
  * The mask is bit-exact: every dropped X_i, read back through ctcb_brnn_activation_offset, is exactly 0 where the
    NumPy mask (tests/net_oracle.py) drops; the first hidden layer is bit-identical to the undropped net's times s
    where it keeps; every activation is within the forward bound of test_configs_gpu.py (1e-4 of the array's largest
    magnitude) of the float64 net with the same mask; the gradient is within 1e-4 per tensor of that net's
    back-propagation through the GPU's own activations, the cost within 1e-4.
  * SGD advances the device counter once per step, inside the CUDA graph: the counter equals SGD.it, the mask in X_i is
    that of step `it`, replays draw new masks and equal eager steps bit for bit, and a toFile / fromFile round trip
    continues the sequence.
  * One call, micro-batches and two emulated shards draw the same mask per utterance.
  * Forward-only calls never drop; check_grad holds with dropout on.
Each comparison prints its measured errors as one JSON line (pytest -s)."""
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel, workspace_activations
from net_oracle import Net, keep_mask, threshold_scale

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COST_TOL, FWD_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-4
D, K = 41, 32


def _kwargs(c):
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make case c (kind bi / uni / dnn)."""
    kind = c.get("kind", "bi")
    return dict(temporalLayer=-1 if kind == "dnn" else c["tl"], numTemporal=c.get("k", 1),
                unidirectional=kind == "uni", reg=c.get("reg", 0.0))


def _net(c, B, p=0.0, seed=33, train=True, maxUtts=None):
    """The GPU net of case c with the parameters of np.random.seed(33)."""
    import nnets.brnnet
    np.random.seed(33)
    nn = nnets.brnnet.NNet(c.get("D", D), c.get("K", K), c["H"], c["N"], c["T"], maxUtts=maxUtts or B,
                           maxLabels=c["L"], train=train, dropout=p, dropoutSeed=seed, **_kwargs(c))
    nn.initParams()
    return nn


def _batch(c, seed=5):
    T, B, L = c["T"], c["B"], c["L"]
    if c.get("ragged"):
        rng = np.random.RandomState(seed)
        lens = [int(x) for x in rng.randint(int(0.6 * T), T + 1, size=B)]
        lens[0] = T
        nlabs = [int(x) for x in rng.randint(max(1, L // 3), L + 1, size=B)]
    else:
        lens, nlabs = [T] * B, [L] * B
    return lens, recipes.synth_batch(c.get("D", D), c.get("K", K), lens, nlabs, seed=33)


def _dropped_layers(nn):
    tl, k = nn.temporalLayer, nn.numTemporal
    return [i for i in range(1, nn.numLayers + 1) if not (tl > 0 and tl <= i < tl + k)]


def _keep(p, seed, step, layer, gs, Tmax, H):
    """[Tmax][B][H] keep mask of a call whose utterances have minibatch indices gs."""
    return np.stack([keep_mask(p, seed, step, layer, g, Tmax, H) for g in gs], axis=1)


# ------------------------------------------------------------------------------------------------ 4. p = 0
P0_CASES = {
    "c2_as_benchmarked": dict(D=41, K=62, H=512, N=2, tl=1, T=200, L=30, B=32),
    "stack_k2": dict(H=96, N=5, tl=2, k=2, T=40, L=8, B=5, reg=1e-2),
    "uni": dict(H=64, N=3, tl=2, T=40, L=8, B=6, kind="uni"),
    "dnn": dict(H=70, N=3, T=40, L=8, B=6, kind="dnn"),
    "ragged": dict(H=256, N=3, tl=2, T=50, L=10, B=7, ragged=True, reg=1e-3),
}


@pytest.mark.parametrize("name", list(P0_CASES))
def test_p0_is_todays_behaviour(name, cuda):
    """The same handle before and after ctcb_brnn_set_dropout(p = 0) and a non-default utterance map: equal launch
    counts, and the bits of the probabilities, costs, skips, gradient, statistics tail and L2 cost."""
    from _ctcb import lib, check, ptr
    c = P0_CASES[name]
    lens, (datas, labelss) = _batch(c)
    nn = _net(c, c["B"])
    batch = nn._batch.pack(datas, labelss).upload()

    def run():
        nn.costAndGradDevice(batch, want_probs=True)          # first use of everything (side stream, modules)
        cuda.cuda.synchronize()
        n0 = lib.ctcb_launch_count()
        nn.costAndGradDevice(batch, want_probs=True)
        cuda.cuda.synchronize()
        return (lib.ctcb_launch_count() - n0, _bits(nn._probs_view(batch.B, batch.Tmax)),
                _bits(nn.grads_ext[:nn.nparams + 6]), _bits(nn._out))

    ref = run()
    step = cuda.zeros(1, dtype=cuda.int64, device="cuda")
    check(lib.ctcb_brnn_set_dropout(nn._h, 0.0, 12345, ptr(step)))
    check(lib.ctcb_brnn_set_dropout_utts(nn._h, 5, 3))
    got = run()
    assert got[0] == ref[0], (got[0], ref[0])
    for a, b in zip(ref[1:], got[1:]):
        assert np.array_equal(a, b)
    # and p > 0 adds exactly one launch per ReLU hidden layer
    check(lib.ctcb_brnn_set_dropout(nn._h, 0.25, 12345, ptr(step)))
    on = run()
    print(json.dumps({"p0_%s" % name: dict(launches=ref[0], launches_p025=on[0])}))
    assert on[0] == ref[0] + len(_dropped_layers(nn))


# ---------------------------------------------------------------------------------- 5 + 6. mask and gradient
CASES = {
    "h512_cluster_bi_ragged": dict(H=512, N=3, tl=2, T=50, L=10, B=6, ragged=True, sweep=1),
    "h1024_tc_bi": dict(H=1024, N=3, tl=2, T=40, L=8, B=8, sweep=2),
    "h70_uni_ragged": dict(H=70, N=3, tl=2, T=30, L=8, B=5, kind="uni", ragged=True),
    "h70_dnn": dict(H=70, N=2, T=30, L=8, B=5, kind="dnn"),
    "h96_stack_k2": dict(H=96, N=5, tl=2, k=2, T=30, L=8, B=4, reg=1e-2),
    "h64_T1": dict(H=64, N=3, tl=2, T=1, L=1, B=4),
    "h64_g_beyond_16_bits": dict(H=64, N=3, tl=2, T=20, L=5, B=4, u0=70000),
}


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("name", list(CASES))
def test_mask_is_bit_exact_and_gradient_matches_float64(name, p, cuda):
    from _ctcb import lib, check
    c = CASES[name]
    B, N, H = c["B"], c["N"], c["H"]
    u0, seed, step = c.get("u0", 0), 2 ** 40 + 77, 2 ** 33 + 5      # both words of the seed; step mod 2^32 counts
    if "sweep" in c:
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_sweep_plan(H, B, 2, plan))
        assert plan[0] == c["sweep"], list(plan)
    lens, (datas, labelss) = _batch(c)
    Tmax = max(lens)
    gs = [u0 + u for u in range(B)]

    ref = _net(c, B)                                   # the same net without dropout: layer 1 before the mask
    batch = ref._batch.pack(datas, labelss).upload()
    ref.costAndGradDevice(batch)
    X1_plain = workspace_activations(ref, B, Tmax)[0, 1]
    del ref

    nn = _net(c, B, p=p, seed=seed)
    nn.dropoutStep.fill_(step)
    batch = nn._batch.pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, u0=u0)
    assert nn.stats.cpu().numpy()[3] == 0
    assert int(nn.dropoutStep.item()) == step           # a training call reads the counter, never moves it
    np.random.seed(33)
    on = Net(c.get("D", D), c.get("K", K), H, N, c["T"], dropout=p, dropoutSeed=seed, **_kwargs(c))
    on.initParams()
    on.dropoutStep = step
    # 6. forward activations and the gradient through the GPU's own activations, against float64
    r = compare(nn, on, datas, labelss, lens, utts=gs)
    X = r["acts"]
    s = threshold_scale(p)[1]

    # 5. the mask, on every row (padded frames included)
    dropped = _dropped_layers(nn)
    assert dropped
    zero_frac = {}
    for i in dropped:
        keep = _keep(p, seed, step, i, gs, Tmax, H)
        assert (X[0, i][~keep] == 0).all(), i
        zero_frac[i] = float((X[0, i] == 0).mean())
        if i == 1:      # layer 1 reads the features: bit for bit the undropped layer times s, or 0
            want = np.where(keep, X1_plain * s, np.float32(0))
            assert np.array_equal(want.view(np.uint32), X[0, 1].view(np.uint32))
    del nn
    cuda.cuda.empty_cache()

    assert np.array_equal(r["skips"], r["skips_given"])
    cost_err, fwd_err, given = r["cost_given"], max(r["fwd"]["X"]), r["grad_given"]
    print(json.dumps({"dropout_%s_p%g" % (name, p): dict(config=c, zero_fraction=zero_frac, cost_rel_err_max=cost_err,
                                                         forward_activation_rel_err_max=fwd_err,
                                                         grad_rel_err_given_gpu_activations_max=max(given))}))
    assert not r["skips"].all()
    assert cost_err <= COST_TOL, cost_err
    assert fwd_err <= FWD_TOL, fwd_err
    assert max(given) <= GRAD_TOL, given


def test_frames_beyond_16_bits(cuda):
    """One 66000-frame utterance of a narrow DNN: frames t >= 2^16 draw their own masks (the counter word holds t
    whole), bit-exact against NumPy on the first layer."""
    c = dict(H=8, N=2, T=66000, L=3, B=1, kind="dnn")
    p, seed, step = 0.5, 9, 3
    lens, (datas, labelss) = _batch(c)
    ref = _net(c, 1)
    batch = ref._batch.pack(datas, labelss).upload()
    ref.costAndGradDevice(batch)
    X1_plain = workspace_activations(ref, 1, c["T"])[0, 1]
    del ref
    nn = _net(c, 1, p=p, seed=seed)
    nn.dropoutStep.fill_(step)
    batch = nn._batch.pack(datas, labelss).upload()
    nn.costAndGradDevice(batch)
    keep = _keep(p, seed, step, 1, [0], c["T"], c["H"])
    want = np.where(keep, X1_plain * threshold_scale(p)[1], np.float32(0))
    acts = workspace_activations(nn, 1, c["T"])
    assert np.array_equal(want.view(np.uint32), acts[0, 1].view(np.uint32))
    assert not np.array_equal(keep[:1000], keep[65536:66536])
    X2 = acts[0, 2]
    assert (X2[~_keep(p, seed, step, 2, [0], c["T"], c["H"])] == 0).all()


# ------------------------------------------------------------------------------------------- 7. graph replay
SGD_NET = dict(H=64, N=3, tl=2, T=60, L=20, B=8)


def _sgd(useGraphs, p=0.2):
    import sgd
    nn = _net(dict(SGD_NET, D=13, K=11), 8, p=p, seed=7)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    return nn, opt


def _corpus():
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    return dict(zip(keys, datas)), dict(zip(keys, [list(map(str, l)) for l in labelss])), keys


def _step_masks_hold(nn, it, B):
    """X_1 and X_3 of the last step hold the masks of step `it` (dropped units 0), not those of step it - 1."""
    ok, other = True, True
    acts = workspace_activations(nn, B, nn._batch.Tmax)
    for i in (1, 3):
        X = acts[0, i]
        Tmax = X.shape[0]
        ok &= bool((X[~_keep(nn.dropout, nn.dropoutSeed, it, i, range(B), Tmax, X.shape[2])] == 0).all())
        other &= bool((X[~_keep(nn.dropout, nn.dropoutSeed, it - 1, i, range(B), Tmax, X.shape[2])] == 0).all())
    return ok and not other


def test_graph_replays_draw_new_masks_and_equal_eager_steps(cuda):
    """Nine SGD steps on SGD.run's own stream: steps replay from their graphs once the two staging buffers have each
    been seen twice.  After every step the counter equals it and X_i holds step it's masks; replays differ from
    each other; the trajectory equals nine eager steps bit for bit."""
    dd, alis, keys = _corpus()
    random.seed(33)
    nn, opt = _sgd(True)
    masks = []
    for _ in range(9):
        opt.run(dd, alis, list(keys), None)
        cuda.cuda.synchronize()
        assert int(nn.dropoutStep.item()) == opt.it
        assert _step_masks_hold(nn, opt.it, 8), opt.it
        masks.append(workspace_activations(nn, 8, nn._batch.Tmax)[0, 1] == 0)
    assert len(opt._graphs) >= 1
    assert not np.array_equal(masks[-1], masks[-2])
    p_g, v_g = nn.params.cpu().numpy(), opt._vflat.cpu().numpy()
    random.seed(33)
    nn_e, opt_e = _sgd(False)
    for _ in range(9):
        opt_e.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    print(json.dumps({"dropout_graph_replay": dict(graphs=len(opt._graphs), costs=list(map(float, opt.costt)))}))
    assert len(opt_e._graphs) == 0 and int(nn_e.dropoutStep.item()) == 9
    assert np.array_equal(p_g, nn_e.params.cpu().numpy()) and np.array_equal(v_g, opt_e._vflat.cpu().numpy())
    # and the mask matters: without dropout the trajectory is another one
    random.seed(33)
    nn_0, opt_0 = _sgd(True, p=0.0)
    for _ in range(3):
        opt_0.run(dd, alis, list(keys), None)
    assert nn_0.dropoutStep is None


def test_to_file_from_file_continues_the_sequence(cuda, tmp_path):
    """Five steps, save (SGD pickle + stack), three more; a fresh net and optimiser loaded from the file make the same
    three steps bit for bit: fromFile sets the counter to it."""
    dd, alis, keys = _corpus()
    random.seed(33)
    nn, opt = _sgd(True)
    for _ in range(5):
        opt.run(dd, alis, list(keys), None)
    f = str(tmp_path / "params.pk")
    with open(f, "wb") as fid:
        opt.toFile(fid)
        nn.toFile(fid)
    state = random.getstate()
    for _ in range(3):
        opt.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    nn2, opt2 = _sgd(True)
    with open(f, "rb") as fid:
        opt2.fromFile(fid)
        nn2.fromFile(fid)
    assert int(nn2.dropoutStep.item()) == opt2.it == 5
    random.setstate(state)
    for _ in range(3):
        opt2.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    assert int(nn2.dropoutStep.item()) == opt2.it == opt.it == 8
    assert np.array_equal(nn.params.cpu().numpy(), nn2.params.cpu().numpy())
    assert np.array_equal(opt._vflat.cpu().numpy(), opt2._vflat.cpu().numpy())


# -------------------------------------------------------------------------------------- 8. however it is split
ACC_NET = dict(D=13, K=11, H=64, N=3, tl=2, T=60, L=20)


def _ragged():
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=7)


@pytest.mark.parametrize("kind", ["bi", "uni", "dnn"])
def test_micro_batches_draw_the_masks_of_one_call(kind, cuda):
    """B = 8 as one call and as 3 + 3 + 2 micro-batches with dropout 0.3: the gradient agrees within the 1e-5 of
    test_accum_gpu.py (one mask per utterance: mismatched masks would differ by far more)."""
    datas, labelss = _ragged()
    c = dict(ACC_NET, kind=kind, reg=1e-2 if kind == "bi" else 0.0)
    out = []
    for maxUtts in (8, 3):
        nn = _net(c, 8, p=0.3, seed=4, maxUtts=maxUtts)
        nn.dropoutStep.fill_(6)
        costs, grad, skips = nn.costAndGradBatch(datas, labelss)
        out.append((costs, skips, [(dw.cpu().numpy(), db.cpu().numpy()) for dw, db in grad]))
    (c1, s1, g1), (c2, s2, g2) = out
    errs = [e for (a, b), (x, y) in zip(g2, g1) for e in (_rel(a, x), _rel(b, y))]
    cost_err = float(np.max(np.abs(c2 - c1) / np.abs(c1)))
    print(json.dumps({"dropout_accum_%s" % kind: dict(grad_rel_err_max=max(errs), cost_rel_err_max=cost_err)}))
    assert np.array_equal(s1, s2)
    assert cost_err <= 1e-6 and max(errs) <= 1e-5, errs


def test_two_shards_summed_equal_the_full_batch(cuda):
    """Two shards emulated on one GPU with (first, stride) = (r, 2), deferred L2, summed, reg*W once: the full batch's
    gradient with the same masks (test_stack_gpu.py's comparison without dropout)."""
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    datas, labelss = _ragged()
    c = dict(ACC_NET, reg=1e-1)
    full = _net(c, 8, p=0.3, seed=4)
    full.dropoutStep.fill_(2)
    full.costAndGradBatch(datas, labelss)
    g_full = full.grads_ext[:full.nparams + 4].clone()
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _net(c, 4, p=0.3, seed=4)
        nn.dropoutStep.fill_(2)
        nn.dropoutShard = (rank, 2)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    cuda.cuda.synchronize()
    a, b = total.cpu().numpy().astype(np.float64), g_full.cpu().numpy().astype(np.float64)
    err = _rel(a[:-4], b[:-4])
    # the same shards with the default map (every rank's utterances numbered from 0) draw other masks
    wrong = None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _net(c, 4, p=0.3, seed=4)
        nn.dropoutStep.fill_(2)
        nn.dropoutShard = (0, 1)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams].clone()
        wrong = part if wrong is None else wrong + part
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(wrong), _ctcb.current_stream()))
    err_wrong = _rel(wrong.cpu().numpy(), b[:-4])
    print(json.dumps({"dropout_two_shards": dict(grad_rel_err=err, grad_rel_err_unmapped_shards=err_wrong)}))
    assert err < 1e-5
    assert err_wrong > 100 * 1e-5
    assert a[-4] == b[-4] == 8 and abs(a[-3] - b[-3]) / abs(b[-3]) < 1e-6 and a[-1] == b[-1] == 0


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
nn = rnnet.NNet(13, 11, 64, 3, 30, temporalLayer=2, reg=1e-3, maxUtts=parallel.per_rank_capacity(8, world),
                maxLabels=10, dropout=0.3, dropoutSeed=5)
nn.initParams()
opt = sgd.SGD(nn, 30, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
for _ in range(3):
    opt.run(dd, alis, list(keys), None)
torch.cuda.synchronize()
assert int(nn.dropoutStep.item()) == opt.it
np.save(os.path.join(sys.argv[1], "params_w%%d_r%%d.npy" %% (world, rank)), nn.params.cpu().numpy())
if world > 1:
    dist.barrier(); dist.destroy_process_group()
'''


def test_two_ranks_draw_the_masks_of_one_gpu(cuda, tmp_path):
    if cuda.cuda.device_count() < 2:
        pytest.skip("two-rank NCCL test of dropout: needs 2 GPUs, %d visible" % cuda.cuda.device_count())
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", "29631", str(script), str(tmp_path)],
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
    print(json.dumps({"dropout_dp2": dict(params_rel_err=err)}))
    assert np.array_equal(p20, p21)
    assert err < 1e-5


# ------------------------------------------------------------------------------ 9. forward-only and determinism
def test_forward_only_calls_never_drop(cuda):
    c = dict(H=64, N=3, tl=2, T=50, L=10, B=6, ragged=True)
    lens, (datas, labelss) = _batch(c)
    outs = []
    for p in (0.0, 0.4):
        nn = _net(c, 6, p=p)
        if p:
            nn.dropoutStep.fill_(3)
            nn.costAndGradBatch(datas, labelss)       # a training call in between changes nothing
        outs.append([x.view(np.uint32) for x in nn.forwardBatch(datas)])
        test = _net(c, 1, p=p, train=False)
        outs[-1].append(test.costAndGrad(datas[0]).view(np.uint32))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_same_seed_and_step_give_the_same_bytes(cuda):
    c = dict(H=64, N=3, tl=2, T=50, L=10, B=6, ragged=True)
    lens, (datas, labelss) = _batch(c)
    snaps = []
    for seed, step in ((5, 3), (5, 3), (6, 3), (5, 4)):
        nn = _net(c, 6, p=0.4, seed=seed)
        nn.dropoutStep.fill_(step)
        nn.costAndGradBatch(datas, labelss)
        snaps.append(_bits(nn.grads_ext[:nn.nparams + 4]))
    assert np.array_equal(snaps[0], snaps[1])
    assert not np.array_equal(snaps[0], snaps[2]) and not np.array_equal(snaps[0], snaps[3])


# ---------------------------------------------------------------------------------------------- 10. check_grad
def test_check_grad_with_dropout(cuda):
    """NNet.check_grad (forward differences in fp32, as test_brnn_gpu.py) with dropout 0.3 on layer 2: costAndGrad
    never advances the counter, so every evaluation sees one mask.  The step is 1e-3, not test_brnn_gpu.py's 1e-2: with
    this mask the cost is curved enough over a 1e-2 step of W1[0, 0] that its forward difference is 0.456 against a
    derivative of 0.836, and the float64 net of tests/net_oracle.py with the same parameters and mask gives the same
    two numbers (0.0122 apart at 1e-3, 0.0012 at 1e-4)."""
    import nnets.brnnet as rnnet
    datas, labelss = recipes.synth_batch(6, 5, [12], [3], seed=4)
    np.random.seed(8)
    nn = rnnet.NNet(6, 5, 8, 2, 12, temporalLayer=1, dropout=0.3)
    nn.initParams()
    pairs = nn.check_grad(datas[0], labelss[0], epsilon=1e-3, maxChecks=2, verbose=False)
    ana = np.array([p[0] for p in pairs]); num = np.array([p[1] for p in pairs])
    assert int(nn.dropoutStep.item()) == 0
    assert np.abs(ana - num).max() < 0.05 * max(1.0, np.abs(ana).max())
