"""GPU tests of the adaptive optimisers (ctcb_adagrad_step_f32, ctcb_adam_step_f32, SGD(optimizer='adagrad' / 'adam'))
on one H100.

  * Each kernel against the float64 rules of tests/optim_oracle.py, element by element:
    |x - x64| <= C * 2^-24 * S (+ 2^-149 where a value is zero or subnormal), S the sum of the magnitudes of the terms
    of x's formula; C (BOUND) is at most 4x the largest ratio measured.  The bound is sharp in t: for t <= 10 the
    oracle evaluated at t - 1 or t + 1 falls outside it, so a frozen or off-by-one step counter fails.
  * A skipped step (n_valid = 0) leaves w and every state bit for bit; a counter below 1 is step 1.
  * Through SGD on a small BRNN: each step's update against the oracle on that step's own gradient (Adam moves every
    element by about alpha*sign(g) at step 1, so two paths whose gradients differ in the last bits are never compared
    with each other); graph replays equal eager steps; toFile / fromFile continues bit for bit (with dropout too, the
    two sharing one counter); micro-batched and empty-shard steps advance the counter once; runNNet end to end; two
    NCCL ranks stay identical.
Each comparison prints its measured ratios as one JSON line (pytest -s)."""
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import optim_oracle as oo
import recipes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = ("adagrad", "adam")
# largest ratio measured on an H100 80GB HBM3 over every case here: AdaGrad 5.29 (r), Adam 6.09 (w, at the C4 count)
BOUND = {"adagrad": 16.0, "adam": 16.0}
ALPHA, MAXG, B1, B2, EPS = 1e-3, 5.0, 0.9, 0.999, 1e-8
C4_PARAMS = 25331756           # ctcb_brnn_param_count of C4 (H=2048, numLayers=5, temporalLayer=3, D=41, K=35)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# -------------------------------------------------------------------------------------------- kernel alone
def _signed_logu(rng, n, lo, hi):
    return (rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(lo, hi, n)).astype(np.float32)


def _inputs(n, seed, rule):
    """w ~ 0.1 N(0, 1); g and m of magnitude 1e-17 .. 1e3, r and v of 1e-34 .. 1e6; exact zeros in each (every term,
    (1-b2) * g_c^2 included, stays a normal float32)."""
    rng = np.random.RandomState(seed)
    w = (0.1 * rng.randn(n)).astype(np.float32)
    g = _signed_logu(rng, n, -17, 3)
    s1 = _signed_logu(rng, n, -17, 3) if rule == "adam" else np.abs(_signed_logu(rng, n, -34, 6))
    s2 = np.abs(_signed_logu(rng, n, -34, 6))
    for a in (w, g, s1, s2):
        a[rng.rand(n) < 0.05] = 0.0
    if n >= 3:
        g[0], s1[1], s2[2] = 0.0, 0.0, 0.0
    return w, g, [s1] if rule == "adagrad" else [s1, s2]


def _kernel(torch, rule, w, g, states, gnorm2, t, n_valid=1.0):
    """One launch on device copies of float32 host arrays; returns (w, states) on the host."""
    from _ctcb import lib, check, ptr
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    w_d, g_d = dev(w), dev(g)
    s_d = [dev(s) for s in states]
    gn = torch.tensor([gnorm2], dtype=torch.float32, device="cuda")
    nv = None if n_valid is None else torch.tensor([n_valid], dtype=torch.float32, device="cuda")
    step = torch.tensor([t], dtype=torch.int64, device="cuda")
    n = w.shape[0]
    if rule == "adagrad":
        check(lib.ctcb_adagrad_step_f32(ptr(w_d), ptr(s_d[0]), ptr(g_d), n, ALPHA, MAXG, ptr(gn), ptr(nv), ptr(step),
                                        None))
    else:
        check(lib.ctcb_adam_step_f32(ptr(w_d), ptr(s_d[0]), ptr(s_d[1]), ptr(g_d), n, ALPHA, B1, B2, EPS, MAXG, ptr(gn),
                                     ptr(nv), ptr(step), None))
    torch.cuda.synchronize()
    assert int(step.item()) == t                       # the kernel reads the counter, never moves it
    return w_d.cpu().numpy(), [s.cpu().numpy() for s in s_d]


def _oracle(rule, w, g, states, gnorm2, t, n_valid=1.0):
    """[(name, x64, S)] of w and the states."""
    if rule == "adagrad":
        o = oo.adagrad_step(w, states[0], g, ALPHA, MAXG, gnorm2, t, n_valid)
        return [("w", o["w"], o["S_w"]), ("r", o["r"], o["S_r"])]
    o = oo.adam_step(w, states[0], states[1], g, ALPHA, B1, B2, EPS, MAXG, gnorm2, t, n_valid)
    return [("w", o["w"], o["S_w"]), ("m", o["m"], o["S_m"]), ("v", o["v"], o["S_v"])]


def _ratios(rule, got, w, g, states, gnorm2, t, n_valid=1.0, S_from=None):
    """{output: max |x - x64| / (2^-24 S + 2^-149)} against the oracle at step t (S of the oracle at S_from, default t)."""
    want = _oracle(rule, w, g, states, gnorm2, t, n_valid)
    S = want if S_from is None else _oracle(rule, w, g, states, gnorm2, S_from, n_valid)
    return {name: oo.error_ratio(x, x64, s[2]) for x, (name, x64, _), s in zip(got, want, S)}


def _gnorm2(clip):
    """Clip off: |g| = 0.6 maxGNorm; on: |g| = 1.37 maxGNorm, c = 0.7299...  (the kernel reads gnorm2, whatever g)."""
    return float(np.float32((1.37 if clip else 0.6) * MAXG) ** 2)


def _grid_n(torch):
    return 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256 + 5     # just over one grid-stride pass


SIZES = ["1", "3", "1023", "1025", "grid+5"]
STEPS = [1, 2, 10, 10 ** 4, 2 ** 31 + 7]


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("rule", RULES)
def test_kernel_matches_float64(rule, size, t, clip, cuda):
    n = _grid_n(cuda) if size == "grid+5" else int(size)
    w, g, states = _inputs(n, seed=n + t % 1000, rule=rule)
    gnorm2 = _gnorm2(clip)
    w1, s1 = _kernel(cuda, rule, w, g, states, gnorm2, t)
    got = [w1] + s1
    r = _ratios(rule, got, w, g, states, gnorm2, t)
    rec = {"ratios": r}
    if t <= 10 and n >= 1023:                          # the bound tells neighbouring steps apart
        for other in (t - 1, t + 1):
            if other >= 1:
                wrong = _ratios(rule, got, w, g, states, gnorm2, other, S_from=t)
                rec["ratio_vs_step_%d" % other] = max(wrong.values())
                assert max(wrong.values()) > BOUND[rule], (other, wrong)
    print(json.dumps({"optim_%s_n%s_t%d_clip%d" % (rule, size, t, clip): rec}))
    assert all(np.isfinite(x).all() for x in got)
    assert max(r.values()) <= BOUND[rule], r


@pytest.mark.parametrize("rule", RULES)
def test_kernel_at_the_c4_parameter_count(rule, cuda):
    """25.3 M parameters, clip on, t = 3; the oracle runs in chunks of 2^22."""
    n = C4_PARAMS
    w, g, states = _inputs(n, seed=4, rule=rule)
    gnorm2 = _gnorm2(True)
    w1, s1 = _kernel(cuda, rule, w, g, states, gnorm2, 3)
    worst = {}
    for a in range(0, n, 1 << 22):
        sl = slice(a, a + (1 << 22))
        r = _ratios(rule, [w1[sl]] + [s[sl] for s in s1], w[sl], g[sl], [s[sl] for s in states], gnorm2, 3)
        worst = {k: max(v, worst.get(k, 0.0)) for k, v in r.items()}
    print(json.dumps({"optim_%s_c4" % rule: worst}))
    assert max(worst.values()) <= BOUND[rule], worst


@pytest.mark.parametrize("rule", RULES)
def test_skipped_step_leaves_everything_bit_for_bit(rule, cuda):
    w, g, states = _inputs(1025, seed=1, rule=rule)
    w1, s1 = _kernel(cuda, rule, w, g, states, _gnorm2(True), 4, n_valid=0.0)
    assert np.array_equal(_bits(w1), _bits(w))
    for a, b in zip(s1, states):
        assert np.array_equal(_bits(a), _bits(b))
    w2, _ = _kernel(cuda, rule, w, g, states, _gnorm2(True), 4, n_valid=None)      # n_valid NULL: a normal step
    assert not np.array_equal(w2, w)


@pytest.mark.parametrize("rule", RULES)
def test_counter_below_one_is_step_one(rule, cuda):
    w, g, states = _inputs(1025, seed=2, rule=rule)
    ref = _kernel(cuda, rule, w, g, states, _gnorm2(False), 1)
    for t in (0, -7, -2 ** 40):
        got = _kernel(cuda, rule, w, g, states, _gnorm2(False), t)
        for a, b in zip([ref[0]] + ref[1], [got[0]] + got[1]):
            assert np.array_equal(_bits(a), _bits(b)), t


# ------------------------------------------------------------------------------------------------- through SGD
NET = dict(D=13, K=11, H=128, N=2, tl=1, T=60, L=12)


def _net(maxUtts=4, p=0.0, reg=1e-3):
    import nnets.brnnet as rnnet
    np.random.seed(33)
    nn = rnnet.NNet(NET["D"], NET["K"], NET["H"], NET["N"], NET["T"], temporalLayer=NET["tl"], reg=reg,
                    maxUtts=maxUtts, maxLabels=NET["L"], dropout=p, dropoutSeed=7)
    nn.initParams()
    return nn


def _opt(nn, rule, batchSize=4):
    import sgd
    return sgd.SGD(nn, NET["T"], alpha=ALPHA, optimizer=rule, momentum=0.9, maxGradNorm=MAXG, batchSize=batchSize,
                   verbose=False)


def _step_data(k, B=4):
    rng = np.random.RandomState(100 + k)
    lens = [int(x) for x in rng.randint(30, NET["T"] + 1, size=B)]
    nlabs = [int(x) for x in rng.randint(3, NET["L"] + 1, size=B)]
    return recipes.synth_batch(NET["D"], NET["K"], lens, nlabs, seed=200 + k)


def _host_states(opt):
    import sgd
    return [opt._flat[name].cpu().numpy() for name in sgd.OPTIMIZERS[opt.optimizer]]


def _check_update(rule, nn, opt, w0, s0, worst):
    """The update just made, against the oracle on the step's own reduced gradient, gnorm^2, counter and n_valid."""
    g = nn.grads.cpu().numpy()
    gnorm2 = float(nn._gnorm2.cpu().numpy()[0])
    n_valid = float(nn.stats.cpu().numpy()[0])
    t = int(opt._step.item())
    assert t == opt.it
    r = _ratios(rule, [nn.params.cpu().numpy()] + _host_states(opt), w0, g, s0, gnorm2, t, n_valid)
    for k, v in r.items():
        worst[k] = max(worst.get(k, 0.0), v)
    assert max(r.values()) <= BOUND[rule], (opt.it, r)
    return np.sqrt(gnorm2) > MAXG


@pytest.mark.parametrize("rule", RULES)
def test_sgd_steps_match_the_oracle_on_their_own_gradient(rule, cuda):
    """Nine eager steps of a H = 128 BRNN (the cluster sweep), B = 4, a new minibatch each step."""
    from _ctcb import lib, check
    plan = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_sweep_plan(NET["H"], 4, 2, plan))
    nn = _net()
    opt = _opt(nn, rule)
    assert opt._step is not None and nn.dropoutStep is None and opt._vflat is None
    worst, clipped = {}, 0
    for k in range(9):
        datas, labels = _step_data(k)
        batch = nn._batch.pack(datas, labels).upload()
        w0, s0 = nn.params.cpu().numpy(), _host_states(opt)
        opt.it += 1
        opt.step_device(batch, opt._momentum_now())
        cuda.cuda.synchronize()
        clipped += _check_update(rule, nn, opt, w0, s0, worst)
        assert not np.array_equal(nn.params.cpu().numpy(), w0)
    print(json.dumps({"optim_sgd_%s" % rule: dict(ratios=worst, clipped_steps=int(clipped), sweep_plan=list(plan))}))


def _corpus():
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 12, 11, 5, 12, 3, 7, 8]
    datas, labelss = recipes.synth_batch(NET["D"], NET["K"], lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    return dict(zip(keys, datas)), dict(zip(keys, [list(map(str, l)) for l in labelss])), keys


def _run(rule, steps, useGraphs=True, p=0.0, seed=33):
    dd, alis, keys = _corpus()
    random.seed(seed)
    nn = _net(maxUtts=8, p=p)
    opt = _opt(nn, rule, batchSize=8)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    return nn, opt


@pytest.mark.parametrize("rule", RULES)
def test_graph_replay_equals_eager_steps(rule, cuda):
    nn_g, opt_g = _run(rule, 9)
    cuda.cuda.synchronize()
    assert len(opt_g._graphs) >= 1 and int(opt_g._step.item()) == opt_g.it == 9
    nn_e, opt_e = _run(rule, 9, useGraphs=False)
    cuda.cuda.synchronize()
    assert len(opt_e._graphs) == 0
    assert np.array_equal(_bits(nn_g.params.cpu().numpy()), _bits(nn_e.params.cpu().numpy()))
    for a, b in zip(_host_states(opt_g), _host_states(opt_e)):
        assert np.array_equal(_bits(a), _bits(b))
    print(json.dumps({"optim_graph_%s" % rule: dict(graphs=len(opt_g._graphs), costs=list(map(float, opt_g.costt)))}))
    assert opt_g.costt == opt_e.costt


@pytest.mark.parametrize("rule,p", [("adam", 0.0), ("adam", 0.2), ("adagrad", 0.0)])
def test_resume_continues_bit_for_bit(rule, p, cuda, tmp_path):
    """Five steps, save (SGD pickle + stack), three more; a fresh net and optimiser loaded from the file make the same
    three steps bit for bit.  With dropout the optimiser reads the dropout counter, and the masks still follow it."""
    dd, alis, keys = _corpus()
    nn, opt = _run(rule, 5, p=p)
    if p:
        assert opt._step is nn.dropoutStep
    f = str(tmp_path / "params.pk")
    with open(f, "wb") as fid:
        opt.toFile(fid)
        nn.toFile(fid)
    state = random.getstate()
    for _ in range(3):
        opt.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    nn2 = _net(maxUtts=8, p=p)
    opt2 = _opt(nn2, rule, batchSize=8)
    with open(f, "rb") as fid:
        opt2.fromFile(fid)
        nn2.fromFile(fid)
    assert int(opt2._step.item()) == opt2.it == 5
    random.setstate(state)
    for _ in range(3):
        opt2.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    assert int(opt2._step.item()) == opt2.it == opt.it == 8
    assert np.array_equal(_bits(nn.params.cpu().numpy()), _bits(nn2.params.cpu().numpy()))
    for a, b in zip(_host_states(opt), _host_states(opt2)):
        assert np.array_equal(_bits(a), _bits(b))
    # a Nesterov optimiser refuses this checkpoint
    import sgd
    with open(f, "rb") as fid, pytest.raises(ValueError, match="nesterov"):
        sgd.SGD(nn2, NET["T"], optimizer="nesterov").fromFile(fid)


@pytest.mark.parametrize("rule", RULES)
def test_micro_batched_step(rule, cuda):
    """Eight utterances through buffers of three (3 + 3 + 2): the counter advances once, and the update matches the
    oracle on the accumulated gradient."""
    import parallel
    nn = _net(maxUtts=3)
    opt = _opt(nn, rule, batchSize=8)
    datas, labels = _step_data(0, B=8)
    worst = {}
    for _ in range(2):
        w0, s0 = nn.params.cpu().numpy(), _host_states(opt)
        opt.it += 1
        opt.step_device_parts(parallel.micro_batches(list(zip(datas, labels)), 3), opt._momentum_now())
        cuda.cuda.synchronize()
        assert float(nn.stats.cpu().numpy()[0]) == 8
        _check_update(rule, nn, opt, w0, s0, worst)
    print(json.dumps({"optim_parts_%s" % rule: worst}))


@pytest.mark.parametrize("rule", RULES)
def test_empty_shard_step_advances_the_counter_once(rule, cuda):
    """A rank with no utterance in the step (emulated on one GPU: the exchange is then a no-op, n_valid = 0): the counter
    advances once, and w and the states keep their bits."""
    nn = _net()
    opt = _opt(nn, rule)
    datas, labels = _step_data(1)
    opt.it += 1
    opt.step_device(nn._batch.pack(datas, labels).upload(), opt._momentum_now())
    w0, s0 = nn.params.cpu().numpy(), _host_states(opt)
    prep = dict(batch=None, pieces=None, used=[], nlab=0, nframes=0)
    opt._launch(prep, None)
    opt._finish(prep, 0)
    cuda.cuda.synchronize()
    assert int(opt._step.item()) == opt.it == 2
    assert np.array_equal(_bits(nn.params.cpu().numpy()), _bits(w0))
    for a, b in zip(_host_states(opt), s0):
        assert np.array_equal(_bits(a), _bits(b))


def test_runnnet_trains_with_adam_and_resumes(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=12, rawsize=20, outputDim=9, T_range=(20, 39), L_range=(3, 8))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--epochs", "2", "--step", "3e-3",
            "--optimizer", "adam", "--beta2", "0.99", "--dataDir", data, "--numFiles", "2", "--inputDim", "16",
            "--rawDim", "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "8", "--save_every", "1",
            "--batchSize", "4", "--runDir", str(tmp_path / "runs"), "--quiet"]
    opt, nn = runNNet.run(args)
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg = load_config(os.path.join(run_dir, "cfg.json"))
    assert (cfg["optimizer"], cfg["beta2"]) == ("adam", 0.99)
    assert opt.optimizer == "adam" and opt.beta2 == 0.99 and int(opt._step.item()) == opt.it == 12
    assert len(opt.costt) == 12 and np.isfinite(opt.costt).all()
    assert np.mean(opt.costt[-3:]) < np.mean(opt.costt[:3])          # it learns
    opt2, nn2 = runNNet.run(["--cfg_file", os.path.join(run_dir, "cfg.json")])
    assert opt2.optimizer == "adam" and opt2.it == opt.it and int(opt2._step.item()) == opt.it
    assert bool((nn2.params == nn.params).all())
    for name in ("moment1", "moment2"):
        assert bool((opt2._flat[name] == opt._flat[name]).all()) and bool(opt._flat[name].abs().sum() > 0)
    out = str(tmp_path / "ll")
    runNNet.run(["--cfg_file", os.path.join(run_dir, "cfg.json"), "--test", "--dataDir", data, "--numFiles", "1",
                 "--outDir", out])
    ark = open(os.path.join(out, "loglikelihoods1.ark"), "rb").read()
    assert ark.startswith(b"utt1_0000 \x00BFM ")


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
                maxLabels=10)
nn.initParams()
opt = sgd.SGD(nn, 30, alpha=1e-3, optimizer="adam", maxGradNorm=5.0, batchSize=8, verbose=False)
for _ in range(4):
    opt.run(dd, alis, list(keys), None)
torch.cuda.synchronize()
assert int(opt._step.item()) == opt.it
out = np.concatenate([nn.params.cpu().numpy(), opt._flat["moment1"].cpu().numpy(), opt._flat["moment2"].cpu().numpy()])
np.save(os.path.join(sys.argv[1], "state_w%%d_r%%d.npy" %% (world, rank)), out)
if world > 1:
    dist.barrier(); dist.destroy_process_group()
'''


def test_two_ranks_stay_identical_under_adam(cuda, tmp_path):
    if cuda.cuda.device_count() < 2:
        pytest.skip("two-rank NCCL test of Adam: needs 2 GPUs, %d visible" % cuda.cuda.device_count())
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", "29641", str(script), str(tmp_path)],
                         env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        _, err = p.communicate(timeout=600)
    finally:
        if p.poll() is None:
            p.kill()
    assert p.returncode == 0, err[-2000:]
    r0, r1 = np.load(tmp_path / "state_w2_r0.npy"), np.load(tmp_path / "state_w2_r1.npy")
    assert np.array_equal(_bits(r0), _bits(r1))
