"""GPU tests of the SpecAugment input masks (ctcb_input_mask_f32, ctcb_brnn_set_input_masks, NNet(freqMasks=...), SGD,
runNNet) on one H100.  A mask either zeroes an element or copies it, so every comparison is bit for bit:

  1. the pass alone against tests/input_mask_oracle.py, with NaN guard bands around its output and feats unchanged;
  2. a masked training call equals an unmasked call of the same net on features masked in NumPy: costs, skips, the
     gradient with its statistics tail, the L2 cost and the probabilities, for ReLU (bi, uni), DNN, stacked, LSTM with
     peepholes, layer norm with dropout and subsampled nets; map 1's contraction plans are the same on both inputs;
  3. micro-batches and emulated shards draw the masks of one call; graph replays draw a new mask each step and equal
     eager steps; toFile / fromFile continues the sequence; check_grad holds;
  4. forward-only calls never mask; counts 0 issue the launches and bits of a net without masks;
  5. forced stalls of either stream keep every output's bytes;
  6. runNNet records the flags, resumes, and resumes an old cfg.json unmasked."""
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import input_mask_oracle as imo
import recipes
from net_check import bits as _bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICY = dict(freqMasks=2, freqMaskWidth=15, timeMasks=2, timeMaskWidth=70, timeMaskRatio=0.2)


def _masked_datas(datas, nu, pol, seed, step, gs):
    """The per-utterance (D x T) features masked as minibatch utterances gs at `step`."""
    out = []
    for d, g in zip(datas, gs):
        D, T = d.shape
        m = imo.batch_mask([T], T, D, nu, pol["freqMasks"], pol["freqMaskWidth"], pol["timeMasks"],
                           pol["timeMaskWidth"], pol["timeMaskRatio"], seed, step, first=g)
        out.append(np.ascontiguousarray(imo.apply(d.T[:, None, :], m)[:, 0, :].T))
    return out


# ------------------------------------------------------------------------------------------------ 1. the pass alone
PASS_CASES = {
    "nu41_c15": dict(nu=41, c=15, lens=[37, 1, 20, 64, 9]),
    "nu41_c1": dict(nu=41, c=1, lens=[70, 3, 41]),
    "nu40_c15_vec": dict(nu=40, c=15, lens=[30, 12, 1]),
    "nu20_c5_vec_straddle": dict(nu=20, c=5, lens=[100, 33, 2, 77]),
    "nu8_c1_vec": dict(nu=8, c=1, lens=[150, 140], pol=dict(POLICY, freqMaskWidth=8)),
    "nu7_c3_odd": dict(nu=7, c=3, lens=[5, 3, 1, 2, 4, 6, 1, 8, 7], pol=dict(POLICY, freqMaskWidth=3)),   # B = 9, D 21
    "B1_long": dict(nu=41, c=3, lens=[300]),
    "wide_masks": dict(nu=13, c=3, lens=[4, 2, 1, 6], pol=dict(freqMasks=64, freqMaskWidth=13, timeMasks=64,
                                                                timeMaskWidth=1000, timeMaskRatio=1.0)),
    "placed": dict(nu=41, c=3, lens=[25, 18, 30], first=2 ** 33 + 3, stride=5, step=2 ** 32 + 9, seed=2 ** 40 + 1),
    "time_only": dict(nu=41, c=15, lens=[60, 45], pol=dict(freqMasks=0, freqMaskWidth=0, timeMasks=3, timeMaskWidth=20,
                                                           timeMaskRatio=0.5)),
    "counts_zero": dict(nu=41, c=3, lens=[10, 7], pol=dict(freqMasks=0, freqMaskWidth=5, timeMasks=0, timeMaskWidth=5,
                                                           timeMaskRatio=1.0)),
}


@pytest.mark.parametrize("name", list(PASS_CASES))
def test_pass_alone_is_the_restatement_bit_for_bit(name, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    c = PASS_CASES[name]
    nu, C, lens = c["nu"], c["c"], c["lens"]
    pol = c.get("pol", POLICY)
    D, B, Tmax = nu * C, len(lens), max(lens) + 3
    first, stride, step, seed = c.get("first", 0), c.get("stride", 1), c.get("step", 11), c.get("seed", 33)
    rng = np.random.RandomState(3)
    x = rng.randn(Tmax, B, D).astype(np.float32)
    x[-1, 0, :] = np.nan                       # padding rows and NaNs are copied as they are
    feats = torch.from_numpy(x).cuda()
    feats_before = _bits(feats)
    guard = 1024                               # NaN guard bands on both sides of the output
    buf = torch.full((2 * guard + x.size,), float("nan"), dtype=torch.float32, device="cuda")
    out = buf[guard:guard + x.size]
    T = torch.tensor(lens, dtype=torch.int32, device="cuda")
    st = torch.tensor([step], dtype=torch.int64, device="cuda")
    check(lib.ctcb_input_mask_f32(ptr(feats), ptr(T), B, Tmax, D, nu, pol["freqMasks"], pol["freqMaskWidth"],
                                  pol["timeMasks"], pol["timeMaskWidth"], pol["timeMaskRatio"], seed, ptr(st), first,
                                  stride, ptr(out), _ctcb.current_stream()))
    torch.cuda.synchronize()
    m = imo.batch_mask(lens, Tmax, D, nu, pol["freqMasks"], pol["freqMaskWidth"], pol["timeMasks"],
                       pol["timeMaskWidth"], pol["timeMaskRatio"], seed, step, first, stride)
    want = imo.apply(x, m)
    got = out.cpu().numpy().reshape(Tmax, B, D)
    g = buf.cpu().numpy()
    print(json.dumps({"input_mask_pass_%s" % name: dict(masked_fraction=float(m.mean()), D=D, B=B, Tmax=Tmax)}))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.isnan(g[:guard]).all() and np.isnan(g[guard + x.size:]).all()
    assert np.array_equal(_bits(feats), feats_before)
    if pol["freqMasks"] + pol["timeMasks"] > 0:
        assert m.any()


# ------------------------------------------------------------------------------------ 2. the step on masked input
D_NU, D_C = 41, 3
STEP_CASES = {
    "bi_relu_ragged": dict(H=64, N=3, tl=2, reg=1e-2),
    "uni_relu": dict(H=64, N=3, tl=2, unidirectional=True),
    "dnn": dict(H=70, N=3, tl=-1),
    "stack_k2": dict(H=96, N=4, tl=1, numTemporal=2, reg=1e-3),
    "lstm_peephole": dict(H=64, N=3, tl=2, cell="lstm", peephole=True),
    "layernorm_dropout": dict(H=64, N=3, tl=2, layerNorm=True, dropout=0.3),
    "subsample_map1": dict(H=64, N=3, tl=2, subsample=2, subsampleLayer=1),
    "subsample_map2": dict(H=64, N=3, tl=2, subsample=2, subsampleLayer=2),
    "c15_wide_input": dict(H=64, N=2, tl=1, nu=41, c=15),
    "c1_vec": dict(H=64, N=2, tl=1, nu=40, c=1),
}


def _step_net(c, B, masks, maxUtts=None, seed=7, **kw):
    import nnets.brnnet
    np.random.seed(33)
    args = dict(c)
    nu, C = args.pop("nu", D_NU), args.pop("c", D_C)
    tl = args.pop("tl")
    extra = dict(POLICY, featDim=nu) if masks else {}
    nn = nnets.brnnet.NNet(nu * C, 11, args.pop("H"), args.pop("N"), 60, temporalLayer=tl, maxUtts=maxUtts or B,
                           maxLabels=12, dropoutSeed=seed, **args, **extra, **kw)
    nn.initParams()
    return nn


def _plan(transA, transB, M, N, K, A, lda, Bp, ldb):
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan(transA, transB, M, N, K, A, lda, Bp, ldb, 1, out))
    return list(out)


def _masked_copy_ptr(nn):
    """The masked copy lies behind everything else in the training workspace."""
    copy = nn.maxBatch * nn.maxUtts * nn.inputDim * 4
    return nn._ws.data_ptr() + nn._ws.numel() - (copy + 255) // 256 * 256


def _outputs(nn, batch):
    nn.costAndGradDevice(batch, want_probs=True)
    nn._torch.cuda.synchronize()
    return (_bits(nn._out), _bits(nn.grads_ext[:nn.nparams + 6]),
            _bits(nn._probs_view(batch.B, nn.frames(batch.Tmax))))


@pytest.mark.parametrize("name", list(STEP_CASES))
def test_step_equals_the_step_on_masked_input(name, cuda):
    c = STEP_CASES[name]
    nu, C = c.get("nu", D_NU), c.get("c", D_C)
    lens = [60, 41, 1, 27, 55, 13]
    datas, labelss = recipes.synth_batch(nu * C, 11, lens, [9, 7, 1, 6, 12, 3], seed=21)
    B, step, u0 = len(lens), 2 ** 32 + 17, 4
    on = _step_net(c, B, True)
    on.dropoutStep.fill_(step)
    off = _step_net(c, B, False)
    if off.dropoutStep is not None:
        off.dropoutStep.fill_(step)
    gs = [u0 + u for u in range(B)]
    b_on = on._batch.pack(datas, labelss).upload()
    b_off = off._batch.pack(_masked_datas(datas, nu, POLICY, 7, step, gs), labelss).upload()
    # map 1 takes the same plans whichever input it reads (the masked copy is 256-byte aligned like feats)
    D, Tmax = nu * C, max(lens)
    k = on.subsample if on.subsample > 1 and on.subsampleLayer == 1 else 1
    if k == 1:
        R, n1, W1 = Tmax * B, on._map_rows(1), on.stack[0][0].data_ptr()
        for A in (_masked_copy_ptr(on), b_off.d_feats.data_ptr()):
            assert _plan(0, 1, R, n1, D, A, D, W1, D) == _plan(0, 1, R, n1, D, b_on.d_feats.data_ptr(), D, W1, D)
            assert _plan(1, 0, n1, D, R, W1, n1, A, D) == _plan(1, 0, n1, D, R, W1, n1, b_on.d_feats.data_ptr(), D)
    on.costAndGradDevice(b_on, want_probs=True, u0=u0)
    cuda.cuda.synchronize()
    got = (_bits(on._out), _bits(on.grads_ext[:on.nparams + 6]), _bits(on._probs_view(B, on.frames(Tmax))))
    # the same u0 places the utterances for dropout too (layernorm_dropout): both nets draw its masks alike
    off.costAndGradDevice(b_off, want_probs=True, u0=u0)
    cuda.cuda.synchronize()
    want = (_bits(off._out), _bits(off.grads_ext[:off.nparams + 6]), _bits(off._probs_view(B, off.frames(Tmax))))
    assert int(on.dropoutStep.item()) == step      # a call reads the counter, never moves it
    assert on.stats.cpu().numpy()[3] == 0 and not on._skip[:B].cpu().numpy().all()
    names = ("costs+skips", "gradient+tail+regcost", "probabilities")
    for n_, a, b in zip(names, got, want):
        assert np.array_equal(a, b), n_
    # and the masks matter: the unmasked features give another gradient
    b_plain = off._batch.pack(datas, labelss).upload()
    off.costAndGradDevice(b_plain, u0=u0)
    cuda.cuda.synchronize()
    assert not np.array_equal(_bits(off.grads_ext[:off.nparams]), want[1][:off.nparams])
    print(json.dumps({"input_mask_step_%s" % name: "bit-identical"}))


def test_counts_zero_is_todays_net(cuda):
    """A net laid out for masks (maskFeatDim > 0) told counts 0: the launches and bits of a net without masks."""
    from _ctcb import lib, check, ptr
    c = STEP_CASES["bi_relu_ragged"]
    lens = [60, 41, 1, 27]
    datas, labelss = recipes.synth_batch(D_NU * D_C, 11, lens, [9, 7, 1, 6], seed=21)
    nets = [_step_net(c, 4, True), _step_net(c, 4, False)]
    check(lib.ctcb_brnn_set_input_masks(nets[0]._h, 0, 0, 0, 0, 1.0, 0, None))
    res = []
    for nn in nets:
        batch = nn._batch.pack(datas, labelss).upload()
        nn.costAndGradDevice(batch, want_probs=True)
        cuda.cuda.synchronize()
        n0 = lib.ctcb_launch_count()
        out = _outputs(nn, batch)
        res.append((lib.ctcb_launch_count() - n0,) + out)
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1:], res[1][1:]):
        assert np.array_equal(a, b)
    # masks on add exactly one launch
    step = cuda.zeros(1, dtype=cuda.int64, device="cuda")
    check(lib.ctcb_brnn_set_input_masks(nets[0]._h, 2, 15, 2, 70, 0.2, 7, ptr(step)))
    batch = nets[0]._batch
    n0 = lib.ctcb_launch_count()
    _outputs(nets[0], batch)
    assert lib.ctcb_launch_count() - n0 == res[1][0] + 1


# ----------------------------------------------------------------------------------------------- 3. invariance
INV_NET = dict(H=64, N=3, tl=2, reg=1e-2)


def _ragged():
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    return recipes.synth_batch(D_NU * D_C, 11, lens, [9, 12, 8, 11, 5, 12, 3, 7], seed=7)


def test_micro_batches_draw_the_masks_of_one_call(cuda):
    """B = 8 in micro-batches of 3 + 3 + 2: bit for bit the same micro-batched net on the features masked as
    minibatch utterances 0..7 of one call."""
    datas, labelss = _ragged()
    on = _step_net(INV_NET, 8, True, maxUtts=3)
    on.dropoutStep.fill_(5)
    off = _step_net(INV_NET, 8, False, maxUtts=3)
    c_on, _, s_on = on.costAndGradBatch(datas, labelss)
    c_off, _, s_off = off.costAndGradBatch(_masked_datas(datas, D_NU, POLICY, 7, 5, range(8)), labelss)
    assert np.array_equal(c_on, c_off) and np.array_equal(s_on, s_off)
    assert np.array_equal(_bits(on.grads_ext[:on.nparams + 6]), _bits(off.grads_ext[:off.nparams + 6]))


def test_two_shards_draw_the_masks_of_one_call(cuda):
    """Rank r of 2 takes utterances r, r + 2, ..: with dropoutShard = (r, 2) its call equals, bit for bit, the unmasked
    net on those utterances masked as minibatch utterances r + 2u."""
    import parallel
    datas, labelss = _ragged()
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        on = _step_net(INV_NET, 4, True)
        on.dropoutStep.fill_(3)
        on.dropoutShard = (rank, 2)
        off = _step_net(INV_NET, 4, False)
        on.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        off.costAndGradBatch(_masked_datas([datas[i] for i in idx], D_NU, POLICY, 7, 3, idx),
                             [labelss[i] for i in idx])
        assert np.array_equal(_bits(on.grads_ext[:on.nparams + 6]), _bits(off.grads_ext[:off.nparams + 6])), rank


def _sgd(useGraphs, masks=True):
    import sgd
    nn = _step_net(dict(H=64, N=3, tl=2), 8, masks)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    return nn, opt


def _corpus():
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 12, 11, 5, 12, 3, 7, 8]
    datas, labelss = recipes.synth_batch(D_NU * D_C, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    return dict(zip(keys, datas)), dict(zip(keys, [list(map(str, l)) for l in labelss])), keys


def _copy_holds_step(nn, it):
    """The masked copy of the last step is the staged batch masked for step `it` (and not for it - 1)."""
    b = nn._batch
    D, B, Tmax = nn.inputDim, b.B, b.Tmax
    n = Tmax * B * D
    off = _masked_copy_ptr(nn) - nn._ws.data_ptr()
    copy = nn._ws[off:off + 4 * n].view(nn._torch.float32).cpu().numpy().reshape(Tmax, B, D)
    x = b.d_feats[:n].cpu().numpy().reshape(Tmax, B, D)
    lens = b.d_lens[:B].cpu().numpy().tolist()
    p = [POLICY[k] for k in ("freqMasks", "freqMaskWidth", "timeMasks", "timeMaskWidth", "timeMaskRatio")]
    want = imo.apply(x, imo.batch_mask(lens, Tmax, D, D_NU, *p, nn.dropoutSeed, it))
    prev = imo.apply(x, imo.batch_mask(lens, Tmax, D, D_NU, *p, nn.dropoutSeed, it - 1))
    return np.array_equal(copy.view(np.uint32), want.view(np.uint32)) and not np.array_equal(copy, prev)


def test_graph_replays_draw_new_masks_and_equal_eager_steps(cuda):
    dd, alis, keys = _corpus()
    random.seed(33)
    nn, opt = _sgd(True)
    for _ in range(9):
        opt.run(dd, alis, list(keys), None)
        cuda.cuda.synchronize()
        assert int(nn.dropoutStep.item()) == opt.it
        assert _copy_holds_step(nn, opt.it), opt.it
    assert len(opt._graphs) >= 1
    p_g, v_g = nn.params.cpu().numpy(), opt._vflat.cpu().numpy()
    random.seed(33)
    nn_e, opt_e = _sgd(False)
    for _ in range(9):
        opt_e.run(dd, alis, list(keys), None)
    cuda.cuda.synchronize()
    assert len(opt_e._graphs) == 0 and int(nn_e.dropoutStep.item()) == 9
    assert np.array_equal(p_g, nn_e.params.cpu().numpy()) and np.array_equal(v_g, opt_e._vflat.cpu().numpy())
    random.seed(33)
    nn_0, opt_0 = _sgd(True, masks=False)
    for _ in range(9):
        opt_0.run(dd, alis, list(keys), None)
    assert nn_0.dropoutStep is None and not np.array_equal(p_g, nn_0.params.cpu().numpy())
    print(json.dumps({"input_mask_graph_replay": dict(graphs=len(opt._graphs), costs=list(map(float, opt.costt)))}))


def test_to_file_from_file_continues_the_sequence(cuda, tmp_path):
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
                maxLabels=10, freqMasks=2, freqMaskWidth=15, timeMasks=2, timeMaskWidth=10, timeMaskRatio=0.2,
                featDim=41)
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
        pytest.skip("two-rank NCCL test of the input masks: needs 2 GPUs, %d visible" % cuda.cuda.device_count())
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", "29633", str(script), str(tmp_path)],
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
    assert np.array_equal(p20, p21)
    assert err < 1e-5


def test_check_grad_with_masks(cuda):
    """costAndGrad never moves the counter, so every evaluation of check_grad sees one mask."""
    import nnets.brnnet as rnnet
    datas, labelss = recipes.synth_batch(15, 5, [12], [3], seed=4)
    np.random.seed(8)
    nn = rnnet.NNet(15, 5, 8, 2, 12, temporalLayer=1, featDim=5, freqMasks=1, freqMaskWidth=2, timeMasks=1,
                    timeMaskWidth=4, timeMaskRatio=0.5)
    nn.initParams()
    nn.dropoutStep.fill_(3)
    pairs = nn.check_grad(datas[0], labelss[0], epsilon=1e-3, maxChecks=3, verbose=False)
    ana = np.array([p[0] for p in pairs])
    num = np.array([p[1] for p in pairs])
    assert int(nn.dropoutStep.item()) == 3
    assert np.abs(ana - num).max() < 0.05 * max(1.0, np.abs(ana).max())


# ----------------------------------------------------------------------------------- 4. forward-only calls
def test_forward_only_calls_never_mask(cuda):
    datas, labelss = _ragged()
    outs = []
    for masks in (False, True):
        nn = _step_net(INV_NET, 8, masks)
        if masks:
            nn.dropoutStep.fill_(3)
            nn.costAndGradBatch(datas, labelss)          # a training call in between changes nothing
        outs.append([x.view(np.uint32) for x in nn.forwardBatch(datas)])
        test = _step_net(INV_NET, 1, masks, train=False)
        outs[-1].append(test.costAndGrad(datas[0]).view(np.uint32))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------- 5. forced stalls
@pytest.mark.parametrize("mode", ["main", "side"])
def test_outputs_keep_their_bytes_under_stalls(mode, cuda):
    """CTCB_STALL holds one stream for a while after each point where the two streams meet: the masked copy must live
    until the side stream's last read, so every output keeps its bytes."""
    from _ctcb import lib, check
    c = dict(H=64, N=3, tl=1, numTemporal=2, reg=1e-3)
    datas, labelss = _ragged()
    nn = _step_net(c, 8, True)
    nn.dropoutStep.fill_(4)
    batch = nn._batch.pack(datas, labelss).upload()
    ref = _outputs(nn, batch)
    try:
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL", mode.encode()))
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL_US", b"2000"))
        got = _outputs(nn, batch)
    finally:
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL", b"off"))
        check(lib.ctcb_debug_set_knob(b"CTCB_STALL_US", None))
    for a, b in zip(ref, got):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------- 6. runNNet
def test_run_nnet_records_the_flags_resumes_and_tests_unmasked(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=15, outputDim=9, T_range=(12, 39), L_range=(2, 5))
    base = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--epochs", "1", "--step", "1e-3",
            "--dataDir", data, "--numFiles", "2", "--inputDim", "15", "--rawDim", "15", "--outputDim", "9",
            "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1", "--quiet"]
    masks = ["--freqMasks", "2", "--freqMaskWidth", "2", "--timeMasks", "2", "--timeMaskWidth", "8",
             "--timeMaskRatio", "0.3", "--featDim", "5"]
    _, net = runNNet.run(base + masks + ["--runDir", str(tmp_path / "runs")])
    assert net.inputMasks and net.featDim == 5 and int(net.dropoutStep.item()) > 0
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert (cfg["freqMasks"], cfg["freqMaskWidth"], cfg["timeMasks"], cfg["timeMaskWidth"], cfg["timeMaskRatio"],
            cfg["featDim"]) == (2, 2, 2, 8, 0.3, 5)
    # resume for a second epoch: the counter continues from it
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    opt2, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.inputMasks and int(net2.dropoutStep.item()) == opt2.it
    # a cfg.json from before the flags resumes unmasked
    old = {k: v for k, v in cfg.items() if k not in ("freqMasks", "freqMaskWidth", "timeMasks", "timeMaskWidth",
                                                      "timeMaskRatio", "featDim")}
    old_dir = str(tmp_path / "old_run")
    os.makedirs(old_dir)
    old.update(output_dir=old_dir, epochs=1)
    dump_config(old, os.path.join(old_dir, "cfg.json"))
    _, net3 = runNNet.run(["--cfg_file", os.path.join(old_dir, "cfg.json"), "--quiet"])
    assert not net3.inputMasks and net3.dropoutStep is None
    # --test writes the same arks from the masked run's cfg.json and from one without the flags
    arks = []
    for cf in (cfg_file, os.path.join(old_dir, "cfg.json")):
        if cf != cfg_file:
            dump_config(dict(old, output_dir=run_dir), cf)
        out = str(tmp_path / ("arks%d" % len(arks)))
        runNNet.run(["--cfg_file", cf, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out])
        arks.append([open(os.path.join(out, f), "rb").read() for f in sorted(os.listdir(out))])
    assert arks[0] and arks[0] == arks[1]
