"""GPU tests of the Gaussian weight noise (ctcb_brnn_weight_noise_f32, ctcb_brnn_set_weight_noise, NNet(weightNoise=..),
SGD, runNNet) on one H100:

  1. the pass alone against tests/weight_noise_oracle.py: every noise term within 1 ulp of the restatement's, every
     other element (alignment gaps included) bit for bit, NaN guard bands around the output, params unchanged, the
     same bits for the same step and new noise for the next; sigma = 0 copies;
  2. a noisy training call equals, bit for bit, an unnoised call of the same net on the noised vector followed by the
     L2 term of the CLEAN weights: costs, skips, every gradient tensor, the statistics tail and the probabilities, for
     bi-directional ReLU on the cluster and on the tensor-core sweep, uni-directional, DNN, stacked, LSTM-peephole,
     layer-norm-with-dropout, subsampled and SpecAugment nets; the L2 cost is the clean net's; params keep their bits;
  3. one SGD step updates the clean weights; micro-batches, emulated shards, graph replays and toFile / fromFile draw
     the noise of one uninterrupted call per step; check_grad holds;
  4. forward-only calls never add noise; sigma = 0 issues the launches and bits of a net without noise;
  5. forced stalls of either stream keep every output's bytes;
  6. runNNet records the flag, resumes, and tests without noise."""
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import recipes
import weight_noise_oracle as wno
from net_check import bits as _bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMA = 0.075
D_IN = 41 * 3


def _net(c, B, noise, maxUtts=None, seed=7, **kw):
    import nnets.brnnet
    np.random.seed(33)
    args = dict(c)
    tl = args.pop("tl")
    D = args.pop("D", D_IN)
    kw.setdefault("weightNoise", SIGMA if noise else 0.0)
    nn = nnets.brnnet.NNet(D, 11, args.pop("H"), args.pop("N"), 60, temporalLayer=tl, maxUtts=maxUtts or B,
                           maxLabels=12, dropoutSeed=seed, **args, **kw)
    nn.initParams()
    return nn


def _ranges(nn):
    """(lo, hi) of the noised matrices: W of every [W, b] pair in front of the [gamma, beta] and [P, dummy] pairs."""
    n = len(nn.stack) - len(nn.normedLayers()) - nn.peepholeEntries()
    base = nn.params.data_ptr()
    return [((w.data_ptr() - base) // 4, (w.data_ptr() - base) // 4 + w.numel()) for w, _ in nn.stack[:n]]


def _noised(nn, params=None):
    """The pass of nn's handle on params (default nn.params) at the counter's current value, as a new tensor."""
    import _ctcb
    from _ctcb import lib, check, ptr
    src = nn.params if params is None else params
    out = nn._torch.empty_like(src)
    check(lib.ctcb_brnn_weight_noise_f32(nn._h, ptr(src), ptr(out), _ctcb.current_stream()))
    return out


def _within_one_ulp(got, w, t):
    """got == w + t' in float32 for t' one of t and its two float32 neighbours."""
    ok = np.zeros(got.shape, dtype=bool)
    for tt in (t, np.nextafter(t, np.float32(-np.inf)), np.nextafter(t, np.float32(np.inf))):
        ok |= (w + tt).view(np.uint32) == got.view(np.uint32)
    return ok


# ------------------------------------------------------------------------------------------------ 1. the pass alone
PASS_CASES = {
    "bi_relu": dict(H=64, N=3, tl=2),
    "uni_stack_k2_odd": dict(H=63, N=4, tl=1, numTemporal=2, unidirectional=True, D=41),
    "dnn": dict(H=70, N=3, tl=-1),
    "lstm_peephole_ln": dict(H=64, N=3, tl=2, cell="lstm", peephole=True, layerNorm=True),
    "subsample_map2": dict(H=65, N=3, tl=2, subsample=3, subsampleLayer=2),
    "wide": dict(H=1024, N=3, tl=2),
}


@pytest.mark.parametrize("name", list(PASS_CASES))
def test_pass_alone_against_the_restatement(name, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    nn = _net(PASS_CASES[name], 2, True)
    P = nn.nparams
    rng = np.random.RandomState(5)
    host = rng.randn(P).astype(np.float32)
    host[3] = -0.0
    host[-1] = np.nan                          # the last tensor's tail: copied as it is
    nn.params.copy_(torch.from_numpy(host))    # the alignment gaps hold values too: they must be copied
    before = _bits(nn.params)
    step = 2 ** 32 + 41
    nn.dropoutStep.fill_(step)
    guard = 1024
    buf = torch.full((2 * guard + P,), float("nan"), dtype=torch.float32, device="cuda")
    out = buf[guard:guard + P]
    check(lib.ctcb_brnn_weight_noise_f32(nn._h, ptr(nn.params), ptr(out), _ctcb.current_stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    ranges = _ranges(nn)
    assert ranges == wno.cfg_ranges(nn._cfg)
    inside = np.zeros(P, dtype=bool)
    exact = 0
    for lo, hi in ranges:
        inside[lo:hi] = True
        t = wno.terms(SIGMA, nn.dropoutSeed, step, lo, hi)
        ok = _within_one_ulp(got[lo:hi], host[lo:hi], t)
        assert ok.all(), (lo, hi, np.flatnonzero(~ok)[:5])
        exact += int(((host[lo:hi] + t).view(np.uint32) == got[lo:hi].view(np.uint32)).sum())
    assert np.array_equal(got.view(np.uint32)[~inside], host.view(np.uint32)[~inside])
    assert (got[inside] != host[inside]).mean() > 0.99
    g = buf.cpu().numpy()
    assert np.isnan(g[:guard]).all() and np.isnan(g[guard + P:]).all()
    assert np.array_equal(_bits(nn.params), before)
    # the same step: the same bits; the next step: new noise
    assert np.array_equal(_bits(_noised(nn)), got.view(np.uint32))
    nn.dropoutStep.fill_(step + 1)
    nxt = _noised(nn).cpu().numpy()
    assert (nxt[inside] != got[inside]).mean() > 0.99
    assert np.array_equal(nxt.view(np.uint32)[~inside], host.view(np.uint32)[~inside])
    # 4-byte accesses (params and out not 16-byte aligned): the same bits as the 16-byte ones
    nn.dropoutStep.fill_(step)
    shifted = torch.empty(P + 1, dtype=torch.float32, device="cuda")
    shifted[1:].copy_(nn.params)
    assert np.array_equal(_bits(_noised(nn, shifted[1:])), got.view(np.uint32))
    # sigma 0: a copy
    check(lib.ctcb_brnn_set_weight_noise(nn._h, 0.0, 0, None))
    assert np.array_equal(_bits(_noised(nn)), before)
    print(json.dumps({"weight_noise_pass_%s" % name: dict(params=P, noised=int(inside.sum()),
                                                          exact_fraction=exact / max(1, int(inside.sum())))}))


# ---------------------------------------------------------------------------- 2. the step on the noised vector
STEP_CASES = {
    "bi_relu_cluster": dict(H=256, N=3, tl=2, reg=1e-2),
    "bi_relu_tc": dict(H=1024, N=2, tl=1, reg=1e-3),
    "uni_relu": dict(H=64, N=3, tl=2, unidirectional=True),
    "dnn": dict(H=70, N=3, tl=-1, reg=1e-2),
    "stack_k2": dict(H=96, N=4, tl=1, numTemporal=2, reg=1e-3),
    "lstm_peephole": dict(H=64, N=3, tl=2, cell="lstm", peephole=True, reg=1e-3),
    "layernorm_dropout": dict(H=64, N=3, tl=2, layerNorm=True, dropout=0.3),
    "subsample": dict(H=64, N=3, tl=2, subsample=2, subsampleLayer=2),
    "specaugment": dict(H=64, N=3, tl=2, freqMasks=2, freqMaskWidth=15, timeMasks=2, timeMaskWidth=20,
                        timeMaskRatio=0.2, featDim=41),
}


def _sweep_kind(H, B):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 16)()
    check(lib.ctcb_debug_sweep_plan(H, B, 2, out))
    return int(out[0])


def _call(nn, batch, u0):
    nn.costAndGradDevice(batch, want_probs=True, u0=u0)
    nn._torch.cuda.synchronize()
    return (_bits(nn._out), _bits(nn.grads_ext[:nn.nparams + 4]), _bits(nn.grads_ext[nn.nparams + 5:nn.nparams + 6]),
            _bits(nn._probs_view(batch.B, nn.frames(batch.Tmax))))


@pytest.mark.parametrize("name", list(STEP_CASES))
def test_step_equals_the_unnoised_step_on_the_noised_vector(name, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    c = STEP_CASES[name]
    lens = [60, 41, 1, 27, 55, 13]
    datas, labelss = recipes.synth_batch(D_IN, 11, lens, [9, 7, 1, 6, 12, 3], seed=21)
    B, step, u0 = len(lens), 2 ** 32 + 17, 4
    if name == "bi_relu_tc":
        assert _sweep_kind(1024, B) == 2
    if name == "bi_relu_cluster":
        assert _sweep_kind(256, B) == 1
    on = _net(c, B, True)
    on.dropoutStep.fill_(step)
    clean = _bits(on.params)
    noisy = _noised(on)
    off = _net(dict(c, reg=0.0), B, False)
    off.params.copy_(noisy)
    if off.dropoutStep is not None:
        off.dropoutStep.fill_(step)
    b_on = on._batch.pack(datas, labelss).upload()
    b_off = off._batch.pack(datas, labelss).upload()
    got = _call(on, b_on, u0)
    assert int(on.dropoutStep.item()) == step      # a call reads the counter, never moves it
    assert np.array_equal(_bits(on.params), clean)  # and never writes params
    assert on.stats.cpu().numpy()[3] == 0 and not on._skip[:B].cpu().numpy().all()
    off.costAndGradDevice(b_off, want_probs=True, u0=u0)
    # the L2 term of the clean weights, with the noisy net's reg, on the unnoised call's gradient
    check(lib.ctcb_brnn_apply_l2_f32(on._h, ptr(on.params), ptr(off.grads), _ctcb.current_stream()))
    cuda.cuda.synchronize()
    want = (_bits(off._out), _bits(off.grads_ext[:off.nparams + 4]),
            _bits(off._probs_view(B, off.frames(b_off.Tmax))))
    for n_, a, b in zip(("costs+skips", "gradient+tail", "probabilities"), (got[0], got[1], got[3]), want):
        assert np.array_equal(a, b), n_
    # the L2 cost is the clean net's: the same net with the noise off, on the same clean params
    check(lib.ctcb_brnn_set_weight_noise(on._h, 0.0, 0, None))
    plain = _call(on, b_on, u0)
    assert np.array_equal(got[2], plain[2])
    if on.reg > 0:
        assert got[2][0] != 0
    # and the noise matters: the clean weights give another gradient
    assert not np.array_equal(plain[1][:on.nparams], got[1][:on.nparams])
    print(json.dumps({"weight_noise_step_%s" % name: "bit-identical"}))


def test_sgd_step_updates_the_clean_weights(cuda):
    """One Nesterov step: the look-ahead w + mom v, the noisy call there, then the update kernel on the CLEAN params
    the look-ahead left, by hand, equals SGD's step bit for bit."""
    import sgd
    import _ctcb
    from _ctcb import lib, check, ptr
    c = dict(H=64, N=3, tl=2, reg=1e-2)
    datas, labelss = recipes.synth_batch(D_IN, 11, [50, 37, 44, 29], [9, 12, 11, 5], seed=3)
    nets = [_net(c, 4, True) for _ in range(2)]
    v0 = cuda.from_numpy(np.random.RandomState(2).randn(nets[0].nparams).astype(np.float32) * 1e-3).cuda()
    mom = 0.9
    opt = sgd.SGD(nets[0], 60, alpha=1e-3, momentum=mom, maxGradNorm=5.0, batchSize=4, verbose=False)
    opt._vflat.copy_(v0)
    nets[0].dropoutStep.fill_(6)
    batch = nets[0]._batch.pack(datas, labelss).upload()
    opt._step_eager(batch, mom)
    # by hand on the twin net
    nn = nets[1]
    v = v0.clone()
    gn2 = cuda.zeros(1, dtype=cuda.float32, device="cuda")
    scratch = cuda.zeros(8192, dtype=cuda.uint8, device="cuda")
    st = _ctcb.current_stream()
    nn.dropoutStep.fill_(7)                         # SGD advances the counter first
    check(lib.ctcb_axpy_f32(ptr(nn.params), ptr(v), mom, nn.nparams, st))
    look = _bits(nn.params)
    nn.costAndGradDevice(nn._batch.pack(datas, labelss).upload())
    cuda.cuda.synchronize()
    assert np.array_equal(_bits(nn.params), look)    # the call left the look-ahead point as it was
    check(lib.ctcb_sumsq_f32(ptr(nn.grads), nn.nparams, ptr(gn2), ptr(scratch), st))
    check(lib.ctcb_sgd_nesterov_step_f32(ptr(nn.params), ptr(v), ptr(nn.grads), nn.nparams, mom, 1e-3, 5.0, ptr(gn2),
                                         ptr(nn.stats), st))
    cuda.cuda.synchronize()
    assert int(nets[0].dropoutStep.item()) == 7
    assert np.array_equal(_bits(nets[0].params), _bits(nn.params))
    assert np.array_equal(_bits(opt._vflat), _bits(v))
    assert np.array_equal(_bits(nets[0].grads), _bits(nn.grads))


# ----------------------------------------------------------------------------------------------- 3. invariance
INV_NET = dict(H=64, N=3, tl=2)


def _ragged():
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    return recipes.synth_batch(D_IN, 11, lens, [9, 12, 8, 11, 5, 12, 3, 7], seed=7)


def test_micro_batches_draw_the_noise_of_one_call(cuda):
    """B = 8 in micro-batches of 3 + 3 + 2: bit for bit the same micro-batched net without noise on the vector noised
    for the step."""
    datas, labelss = _ragged()
    on = _net(INV_NET, 8, True, maxUtts=3)
    on.dropoutStep.fill_(5)
    off = _net(INV_NET, 8, False, maxUtts=3)
    off.params.copy_(_noised(on))
    c_on, _, s_on = on.costAndGradBatch(datas, labelss)
    c_off, _, s_off = off.costAndGradBatch(datas, labelss)
    assert np.array_equal(c_on, c_off) and np.array_equal(s_on, s_off)
    assert np.array_equal(_bits(on.grads_ext[:on.nparams + 4]), _bits(off.grads_ext[:off.nparams + 4]))


def test_two_shards_draw_the_noise_of_one_call(cuda):
    """Rank r of 2 takes utterances r, r + 2, ..: its call sees the same noisy weights as any other rank."""
    import parallel
    datas, labelss = _ragged()
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        on = _net(INV_NET, 4, True)
        on.dropoutStep.fill_(3)
        on.dropoutShard = (rank, 2)
        off = _net(INV_NET, 4, False)
        off.params.copy_(_noised(on))
        on.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        off.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        assert np.array_equal(_bits(on.grads_ext[:on.nparams + 4]), _bits(off.grads_ext[:off.nparams + 4])), rank


def _sgd(useGraphs, noise=True, optimizer="adam"):
    import sgd
    nn = _net(dict(INV_NET), 8, noise)
    opt = sgd.SGD(nn, 60, alpha=1e-3, optimizer=optimizer, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    return nn, opt


def _corpus():
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 12, 11, 5, 12, 3, 7, 8]
    datas, labelss = recipes.synth_batch(D_IN, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    return dict(zip(keys, datas)), dict(zip(keys, [list(map(str, l)) for l in labelss])), keys


def _copy(nn):
    """The noisy copy of the last training call: behind everything else in the training workspace."""
    n = (4 * nn.nparams + 255) // 256 * 256
    return _bits(nn._ws[nn._ws.numel() - n:nn._ws.numel() - n + 4 * nn.nparams].view(nn._torch.float32))


def test_graph_replays_draw_new_noise_and_equal_eager_steps(cuda):
    """Adam (no look-ahead): the copy of step `it` is the step's starting params noised for `it`, and not for it - 1."""
    dd, alis, keys = _corpus()
    random.seed(33)
    nn, opt = _sgd(True)
    for _ in range(9):
        p = nn.params.clone()
        opt.run(dd, alis, list(keys), None)
        cuda.cuda.synchronize()
        assert int(nn.dropoutStep.item()) == opt.it
        assert np.array_equal(_copy(nn), _bits(_noised(nn, p))), opt.it
        nn.dropoutStep.fill_(opt.it - 1)
        assert not np.array_equal(_copy(nn), _bits(_noised(nn, p)))
        nn.dropoutStep.fill_(opt.it)
    assert len(opt._graphs) >= 1
    p_g = nn.params.cpu().numpy()
    random.seed(33)
    nn_e, opt_e = _sgd(False)
    for _ in range(9):
        opt_e.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    assert len(opt_e._graphs) == 0 and int(nn_e.dropoutStep.item()) == 9
    assert np.array_equal(p_g, nn_e.params.cpu().numpy())
    for name in ("moment1", "moment2"):
        assert np.array_equal(opt._flat[name].cpu().numpy(), opt_e._flat[name].cpu().numpy())
    random.seed(33)
    nn_0, opt_0 = _sgd(True, noise=False)
    for _ in range(9):
        opt_0.run(dd, alis, list(keys), None)
    assert not np.array_equal(p_g, nn_0.params.cpu().numpy())
    print(json.dumps({"weight_noise_graph_replay": dict(graphs=len(opt._graphs), costs=list(map(float, opt.costt)))}))


def test_to_file_from_file_continues_the_sequence(cuda, tmp_path):
    dd, alis, keys = _corpus()
    random.seed(33)
    nn, opt = _sgd(True, optimizer="nesterov")
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
    nn2, opt2 = _sgd(True, optimizer="nesterov")
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
datas, labelss = recipes.synth_batch(123, 11, lens, [6, 8, 4, 9, 5, 7, 3, 8], seed=9)
keys = ["k%%d" %% i for i in range(len(lens))]
dd = dict(zip(keys, datas)); alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
np.random.seed(2); random.seed(33)
nn = rnnet.NNet(123, 11, 64, 3, 30, temporalLayer=2, reg=1e-3, maxUtts=parallel.per_rank_capacity(8, world),
                maxLabels=10, weightNoise=0.075)
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


def test_two_ranks_draw_the_noise_of_one_gpu(cuda, tmp_path):
    if cuda.cuda.device_count() < 2:
        pytest.skip("two-rank NCCL test of the weight noise: needs 2 GPUs, %d visible" % cuda.cuda.device_count())
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", "29643", str(script), str(tmp_path)],
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
    assert np.array_equal(p20, p21)
    assert float(np.linalg.norm(p20 - p1) / np.linalg.norm(p1)) < 1e-5


def test_check_grad_with_noise(cuda):
    """costAndGrad never moves the counter and the noise does not depend on the weights' values, so check_grad holds:
    the gradient is that of the cost at the noisy weights."""
    import nnets.brnnet as rnnet
    datas, labelss = recipes.synth_batch(15, 5, [12], [3], seed=4)
    np.random.seed(8)
    nn = rnnet.NNet(15, 5, 8, 2, 12, temporalLayer=1, weightNoise=0.05)
    nn.initParams()
    nn.dropoutStep.fill_(3)
    pairs = nn.check_grad(datas[0], labelss[0], epsilon=1e-3, maxChecks=3, verbose=False)
    ana = np.array([p[0] for p in pairs])
    num = np.array([p[1] for p in pairs])
    assert int(nn.dropoutStep.item()) == 3
    assert np.abs(ana - num).max() < 0.05 * max(1.0, np.abs(ana).max())


# ----------------------------------------------------------------------------------- 4. forward-only calls
def test_forward_only_calls_never_add_noise(cuda):
    datas, labelss = _ragged()
    outs = []
    for noise in (False, True):
        nn = _net(INV_NET, 8, noise)
        if noise:
            nn.dropoutStep.fill_(3)
            nn.costAndGradBatch(datas, labelss)          # a training call in between changes nothing
        outs.append([x.view(np.uint32) for x in nn.forwardBatch(datas)])
        test = _net(INV_NET, 1, noise, train=False)
        outs[-1].append(test.costAndGrad(datas[0]).view(np.uint32))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_sigma_zero_is_todays_net(cuda):
    """A net laid out for noise (weightNoise = 1) told sigma 0 issues the launches and bits of a net without it; noise on
    adds exactly one launch.  NNet refuses a negative or non-finite sigma and lays nothing out for sigma 0."""
    from _ctcb import lib, check
    c = dict(H=64, N=3, tl=2, reg=1e-2)
    datas, labelss = recipes.synth_batch(D_IN, 11, [60, 41, 1, 27], [9, 7, 1, 6], seed=21)
    nets = [_net(c, 4, True), _net(c, 4, False)]
    assert nets[1].dropoutStep is None and nets[1]._cfg.weightNoise == 0 and nets[0]._cfg.weightNoise == 1
    check(lib.ctcb_brnn_set_weight_noise(nets[0]._h, 0.0, 0, None))
    res = []
    for nn in nets:
        batch = nn._batch.pack(datas, labelss).upload()
        _call(nn, batch, 0)
        n0 = lib.ctcb_launch_count()
        out = _call(nn, batch, 0)
        res.append((lib.ctcb_launch_count() - n0,) + out)
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1:], res[1][1:]):
        assert np.array_equal(a, b)
    check(lib.ctcb_brnn_set_weight_noise(nets[0]._h, SIGMA, 7, nets[0].dropoutStep.data_ptr()))
    n0 = lib.ctcb_launch_count()
    _call(nets[0], nets[0]._batch, 0)
    assert lib.ctcb_launch_count() - n0 == res[1][0] + 1
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="weightNoise"):
            _net(c, 4, False, weightNoise=bad)
    assert (lib.ctcb_brnn_workspace_bytes(ctypes.byref(nets[1]._cfg)) == nets[1]._ws.numel()
            < nets[0]._ws.numel())


# ------------------------------------------------------------------------------------------- 5. forced stalls
@pytest.mark.parametrize("mode", ["main", "side"])
def test_outputs_keep_their_bytes_under_stalls(mode, cuda):
    """CTCB_STALL holds one stream for a while after each point where the two streams meet: every stage that reads a
    weight must see the noisy copy of this call, so every output keeps its bytes."""
    from _ctcb import lib, check
    c = dict(H=64, N=3, tl=1, numTemporal=2, reg=1e-3)
    datas, labelss = _ragged()
    nn = _net(c, 8, True)
    nn.dropoutStep.fill_(4)
    batch = nn._batch.pack(datas, labelss).upload()
    ref = _call(nn, batch, 0)
    try:
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL", mode.encode()))
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL_US", b"2000"))
        got = _call(nn, batch, 0)
    finally:
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL", b"off"))
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL_US", None))
    for a, b in zip(ref, got):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------- 6. runNNet
def test_run_nnet_records_the_flag_resumes_and_tests_without_noise(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=15, outputDim=9, T_range=(12, 39), L_range=(2, 5))
    base = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--epochs", "1", "--step", "1e-3",
            "--dataDir", data, "--numFiles", "2", "--inputDim", "15", "--rawDim", "15", "--outputDim", "9",
            "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1", "--quiet"]
    _, net = runNNet.run(base + ["--weightNoise", "0.075", "--runDir", str(tmp_path / "runs")])
    assert net.weightNoise == 0.075 and int(net.dropoutStep.item()) > 0
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["weightNoise"] == 0.075
    # resume for a second epoch: the counter continues from it
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    opt2, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.weightNoise == 0.075 and int(net2.dropoutStep.item()) == opt2.it
    # a cfg.json from before the flag resumes without noise
    old = {k: v for k, v in cfg.items() if k != "weightNoise"}
    old_dir = str(tmp_path / "old_run")
    os.makedirs(old_dir)
    old.update(output_dir=old_dir, epochs=1)
    dump_config(old, os.path.join(old_dir, "cfg.json"))
    _, net3 = runNNet.run(["--cfg_file", os.path.join(old_dir, "cfg.json"), "--quiet"])
    assert net3.weightNoise == 0.0 and net3.dropoutStep is None
    # --test writes the same arks from the noisy run's cfg.json and from one without the flag
    arks = []
    for cf in (cfg_file, os.path.join(old_dir, "cfg.json")):
        if cf != cfg_file:
            dump_config(dict(old, output_dir=run_dir), cf)
        out = str(tmp_path / ("arks%d" % len(arks)))
        net_t = runNNet.run(["--cfg_file", cf, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out])
        assert net_t.weightNoise == 0.0 and net_t.dropoutStep is None
        arks.append([open(os.path.join(out, f), "rb").read() for f in sorted(os.listdir(out))])
    assert arks[0] and arks[0] == arks[1]
