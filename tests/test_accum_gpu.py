"""GPU tests of gradient accumulation over micro-batches (ctcb_brnn_cost_and_grad_part, NNet.costAndGradBatch /
SGD with more utterances than the net's buffers hold).

A step computed as several micro-batches must give the gradient of one call on the whole step: the per-utterance
costs and skip flags, the exact utterance counts of the statistics tail, and every gradient tensor up to fp32
summation order (1e-5 relative, Frobenius norm).  Each comparison prints its measured errors (pytest -s)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import recipes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAD_TOL, NLL_TOL = 1e-5, 1e-6


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nb = np.linalg.norm(b)
    if nb == 0.0:
        return 0.0 if np.linalg.norm(a) == 0.0 else float("inf")
    return float(np.linalg.norm(a - b) / nb)


def _make_net(kind, maxUtts, D=13, K=11, H=64, N=3, tl=2, T=60, L=20, reg=0.0):
    import nnets.brnnet
    import nnets.nnet
    import nnets.rnnet
    np.random.seed(4)
    if kind == "bi":
        nn = nnets.brnnet.NNet(D, K, H, N, T, temporalLayer=tl, reg=reg, maxUtts=maxUtts, maxLabels=L)
        assert nn.temporalLayer == tl
    elif kind == "uni":
        nn = nnets.rnnet.NNet(D, K, H, N, T, temporalLayer=tl, maxUtts=maxUtts, maxLabels=L)
    else:
        nn = nnets.nnet.NNet(D, K, H, N, T, maxUtts=maxUtts, maxLabels=L)
    nn.initParams()
    return nn


def _run(nn, datas, labelss):
    costs, grad, skips = nn.costAndGradBatch(datas, labelss)
    g = [(dw.cpu().numpy().astype(np.float64), db.cpu().numpy().astype(np.float64)) for dw, db in grad]
    tail = nn.grads_ext[nn.nparams:nn.nparams + 4].cpu().numpy().astype(np.float64)
    return costs, skips, g, tail, nn.regcost


def _compare(name, full, split, grad_tol=GRAD_TOL):
    """full / split: _run results of one call on the whole step and of the accumulated micro-batches."""
    (c1, s1, g1, t1, r1), (c2, s2, g2, t2, r2) = full, split
    assert np.array_equal(s1, s2), (s1, s2)
    ok = ~s1
    cost_err = float(np.max(np.abs(c2[ok] - c1[ok]) / np.abs(c1[ok])))
    grad_errs = []
    for (dw1, db1), (dw2, db2) in zip(g1, g2):
        grad_errs += [_rel(dw2, dw1), _rel(db2, db1)]
    nll_err = abs(t2[1] - t1[1]) / abs(t1[1])
    print(json.dumps({name: dict(cost_rel_err_max=cost_err, nll_sum_rel_err=nll_err, grad_rel_err_max=max(grad_errs),
                                 grad_rel_err=grad_errs, n_valid=t2[0], n_skipped=t2[2], regcost=(r1, r2))}))
    assert cost_err <= NLL_TOL, cost_err
    assert t2[0] == t1[0] == ok.sum() and t2[2] == t1[2] == (~ok).sum() and t2[3] == t1[3] == 0
    assert nll_err <= NLL_TOL, nll_err
    assert r2 == r1
    assert max(grad_errs) <= grad_tol, grad_errs
    return grad_errs


def _ragged_batch(D=13, K=11, seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    datas, labelss = recipes.synth_batch(D, K, lens, nlabs, seed=seed)
    return datas, labelss


# ---------------------------------------------------------------------------------------------- 1. one big batch
@pytest.mark.parametrize("kind,reg", [("bi", 0.0), ("uni", 0.0), ("ff", 0.0), ("bi", 1e-2)])
def test_accumulated_micro_batches_equal_one_batch(kind, reg, cuda):
    """B = 8 as one call (maxUtts = 8) and as 3 + 3 + 2 (maxUtts = 3), same parameters."""
    datas, labelss = _ragged_batch()
    full = _run(_make_net(kind, 8, reg=reg), datas, labelss)
    split_net = _make_net(kind, 3, reg=reg)
    split = _run(split_net, datas, labelss)
    _compare("%s_reg%g" % (kind, reg), full, split)
    if reg > 0:
        assert split[4] > 0


def test_accumulated_ragged_batch_with_an_infeasible_utterance(cuda):
    """Utterance 2 cannot be aligned (8 repetitions of one label need 15 frames, it has 12): it is skipped in both
    runs, contributes no gradient, and the counts of the tail still add up over the micro-batches."""
    datas, labelss = _ragged_batch()
    labelss[2] = np.full(8, 3, dtype=np.int32)
    full = _run(_make_net("bi", 8, reg=1e-3), datas, labelss)
    split = _run(_make_net("bi", 3, reg=1e-3), datas, labelss)
    assert full[1].sum() == 1 and full[1][2]
    _compare("bi_ragged_infeasible", full, split)


# ------------------------------------------------------------------------- 2. split-K / tensor-core coverage
def test_accumulated_tensor_core_split_k_contractions(cuda):
    """H = 1024, T = 300: every micro-batch of 8 has R = 2400 > 2048 rows, so its H x H weight gradients (and the
    32-row output layer's) run on the tensor-core GEMM with split-K and the deterministic reduce, adding into the
    gradient (beta = 1); the one batch of 24 is the reference.  The recurrences run on the tensor-core sweep.

    Bound 2e-5 instead of 1e-5: here the two sides are not the same sums in another order.  The tensor cores truncate
    their fp32 accumulation (DESIGN.md, numerics), so a 3xTF32 contraction carries an error of a few 1e-6 that grows
    with the accumulator chain: the batch of 24 sums its 7200 rows in 4 chains of 1824, each micro-batch its 2400 rows
    in 3 chains of 800.  The output layer's forward contraction is split differently too (logits, hence costs, differ
    by ~2e-7).  Measured on an H100 80GB HBM3: 1.45e-5 for the 1024 x 1024 dW of the second layer, 1.05e-5 and
    1.12e-5 for the two recurrent matrices, at most 2.7e-6 for the other tensors."""
    D, K, H, N, tl, T, L = 41, 32, 1024, 2, 1, 300, 40
    rng = np.random.RandomState(3)
    lens = [T] + [int(x) for x in rng.randint(200, T + 1, size=23)]
    nlabs = [int(x) for x in rng.randint(10, L + 1, size=24)]
    datas, labelss = recipes.synth_batch(D, K, lens, nlabs, seed=5)
    from _ctcb import lib
    assert lib.ctcb_sweep_uses_tensor_cores(H, 8) == 1
    full = _run(_make_net("bi", 24, D=D, K=K, H=H, N=N, tl=tl, T=T, L=L, reg=1e-3), datas, labelss)
    cuda.cuda.empty_cache()
    split = _run(_make_net("bi", 8, D=D, K=K, H=H, N=N, tl=tl, T=T, L=L, reg=1e-3), datas, labelss)
    _compare("tc_split_k_h1024", full, split, grad_tol=2e-5)


@pytest.mark.parametrize("M,N,K", [(256, 256, 4100),      # tensor cores, split-K + reduce
                                   (1024, 1024, 200),     # tensor cores, direct epilogue
                                   (62, 512, 3000),       # the output layer's gradient on the tensor cores
                                   (11, 64, 3000),        # FFMA kernel, split-K + reduce
                                   (11, 64, 100)])        # FFMA kernel, direct epilogue
@pytest.mark.parametrize("ta,tb", [(1, 0), (0, 1), (0, 0), (1, 1)])
def test_gemm_beta_one_adds_into_c_on_every_path(M, N, K, ta, tb, cuda):
    """C = A.B + C (beta = 1), the weight-gradient contraction of a later micro-batch, on each path ctcb_gemm_f32 can
    take, with every operand orientation; beta = 0 ignores a NaN-filled C."""
    import _ctcb
    from _ctcb import lib, check, ptr
    torch = cuda
    rng = np.random.RandomState(M + N + K + 10 * ta + tb)
    a = rng.randn(M, K).astype(np.float32)
    b = rng.randn(K, N).astype(np.float32)
    c0 = rng.randn(M, N).astype(np.float32)
    A = torch.from_numpy(np.ascontiguousarray(a.T if ta else a)).cuda()
    Bm = torch.from_numpy(np.ascontiguousarray(b.T if tb else b)).cuda()
    lda, ldb = (M if ta else K), (K if tb else N)
    ws = torch.empty(max(1, lib.ctcb_gemm_workspace_bytes(M, N, K)), dtype=torch.uint8, device="cuda")
    st = _ctcb.current_stream()
    want = a.astype(np.float64) @ b.astype(np.float64)
    C = torch.from_numpy(c0.copy()).cuda()
    check(lib.ctcb_gemm_f32(ta, tb, M, N, K, 1.0, ptr(A), lda, ptr(Bm), ldb, 1.0, ptr(C), N, None, 0, None,
                            ptr(ws), ws.numel(), st))
    C0 = torch.full((M, N), float("nan"), device="cuda")
    check(lib.ctcb_gemm_f32(ta, tb, M, N, K, 1.0, ptr(A), lda, ptr(Bm), ldb, 0.0, ptr(C0), N, None, 0, None,
                            ptr(ws), ws.numel(), st))
    torch.cuda.synchronize()
    got, got0 = C.cpu().numpy(), C0.cpu().numpy()
    err1, err0 = _rel(got, want + c0), _rel(got0, want)
    # the sum with C is the product's epilogue: adding C afterwards to the beta = 0 result gives the same bits
    same = np.array_equal(got, got0 + c0)
    print(json.dumps({"gemm_beta_%dx%dx%d_t%d%d" % (M, N, K, ta, tb): dict(beta1=err1, beta0=err0, same_bits=same)}))
    assert np.isfinite(got0).all()
    assert err1 < 1e-5 and err0 < 1e-5
    assert same


# ------------------------------------------------------------------------------------------ 3. ABI contract
def _call(nn, batch, flags, cost=None, skip=None):
    import _ctcb
    from _ctcb import lib, check, ptr
    B = batch.B
    cost = nn._cost[:B] if cost is None else cost
    skip = nn._skip[:B] if skip is None else skip
    args = [nn._h, ptr(batch.d_feats), ptr(batch.d_lens), ptr(batch.d_labels), ptr(batch.d_off), B, batch.Tmax,
            ptr(nn.params), ptr(nn.grads), ptr(cost), ptr(skip), ptr(nn._regcost), None, ptr(nn.stats)]
    tail = [ptr(nn._ws), nn._ws.numel(), _ctcb.current_stream()]
    if flags is None:
        check(lib.ctcb_brnn_cost_and_grad(*(args + tail)))
    else:
        check(lib.ctcb_brnn_cost_and_grad_part(*(args + [flags] + tail)))


def _poison(nn):
    """NaN into every gradient tensor, the statistics tail and the L2 cost (the alignment gaps between tensors of
    the flat vector belong to no tensor and are never written; they stay zero)."""
    for w, b in nn.grad:
        w.fill_(float("nan"))
        b.fill_(float("nan"))
    nn.stats.fill_(float("nan"))
    nn._regcost.fill_(float("nan"))


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


def _snapshot(nn, B):
    """Bits of everything a training call writes: gradient + statistics tail, L2 cost, per-utterance cost and skip."""
    P = nn.nparams
    return (_bits(nn.grads_ext[:P + 4]), _bits(nn.grads_ext[P + 5:P + 6]), _bits(nn._out[:B]),
            _bits(nn._out[nn.maxUtts:nn.maxUtts + B]))


def test_part_first_last_is_bit_identical_to_cost_and_grad(cuda):
    """..._part(FIRST | LAST) = ctcb_brnn_cost_and_grad: same bits and the same number of launches, and FIRST
    ignores a NaN-filled gradient and statistics tail."""
    from _ctcb import lib, PART_FIRST, PART_LAST
    datas, labelss = _ragged_batch()
    nn = _make_net("bi", 8, reg=1e-2)
    batch = nn._batch.pack(datas, labelss).upload()
    _call(nn, batch, None)                    # first use (side stream, module loads)
    n0 = lib.ctcb_launch_count()
    _call(nn, batch, None)
    n_plain = lib.ctcb_launch_count() - n0
    ref = _snapshot(nn, 8)
    _poison(nn)
    nn._out.fill_(float("nan"))
    n0 = lib.ctcb_launch_count()
    _call(nn, batch, PART_FIRST | PART_LAST)
    n_part = lib.ctcb_launch_count() - n0
    got = _snapshot(nn, 8)
    assert n_part == n_plain
    for r, g in zip(ref, got):
        assert np.array_equal(r, g)


def test_repeated_split_is_bit_identical_and_first_ignores_nan(cuda):
    datas, labelss = _ragged_batch()
    nn = _make_net("bi", 3, reg=1e-2)
    P = nn.nparams
    state = lambda: (_bits(nn.grads_ext[:P + 4]), _bits(nn.grads_ext[P + 5:P + 6]))     # noqa: E731
    nn.costAndGradBatch(datas, labelss)
    a = state()
    costs_a, _, skips_a = nn.costAndGradBatch(datas, labelss)
    b = state()
    _poison(nn)
    costs_c, _, skips_c = nn.costAndGradBatch(datas, labelss)
    c = state()
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and all(np.array_equal(x, y) for x, y in zip(a, c))
    assert np.array_equal(costs_a, costs_c) and np.array_equal(skips_a, skips_c)
    assert np.isfinite(nn.grads_ext[:P + 4].cpu().numpy()).all()


def test_error_flag_of_a_middle_part_survives_to_the_tail(cuda):
    """The statistics tail after FIRST and a middle part holds a raised sweep error flag (set by hand here: the
    kernels raise it only on an inter-CTA wait timeout); the LAST part adds into the tail and keeps it, and the
    next step's FIRST clears it."""
    from _ctcb import PART_FIRST, PART_LAST
    datas, labelss = _ragged_batch()
    nn = _make_net("bi", 3, reg=1e-2)
    pieces = [list(range(0, 3)), list(range(3, 6)), list(range(6, 8))]
    for k, idx in enumerate(pieces):
        batch = nn.swap_batches().pack([datas[i] for i in idx], [labelss[i] for i in idx]).upload()
        _call(nn, batch, (PART_FIRST if k == 0 else 0) | (PART_LAST if k == 2 else 0))
        if k == 1:
            nn.stats[3:4].fill_(1.0)
    tail = nn.stats.cpu().numpy()
    assert tail[3] == 1.0 and tail[0] + tail[2] == 8
    with pytest.raises(RuntimeError):        # what a caller reading the tail then does
        nn._rec_host.copy_(nn.record)
        nn._read_record()
    batch = nn.swap_batches().pack(datas[:3], labelss[:3]).upload()
    _call(nn, batch, PART_FIRST | PART_LAST)
    tail = nn.stats.cpu().numpy()
    assert tail[3] == 0.0 and tail[0] + tail[2] == 3


def test_unknown_flags_are_rejected(cuda):
    datas, labelss = _ragged_batch()
    nn = _make_net("bi", 8)
    batch = nn._batch.pack(datas, labelss).upload()
    with pytest.raises(ValueError):
        _call(nn, batch, 4)


# ------------------------------------------------------------------------------------ 4. optimiser trajectory
def _train(maxUtts, batchSize, lens, nlabs, steps, useGraphs=True, reg=1e-2):
    import random
    import nnets.brnnet
    import sgd
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    np.random.seed(2)
    random.seed(33)
    nn = nnets.brnnet.NNet(13, 11, 64, 3, max(lens), temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20)
    nn.initParams()
    opt = sgd.SGD(nn, max(lens), alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=batchSize, verbose=False)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    import torch
    torch.cuda.synchronize()
    return (nn.params.cpu().numpy().astype(np.float64), opt._vflat.cpu().numpy().astype(np.float64),
            np.array(opt.costt), opt)


def test_sgd_accumulated_steps_follow_the_single_batch_trajectory(cuda):
    """batchSize = 8 on maxUtts = 3 (three micro-batches per step, run eagerly) against maxUtts = 8 (one call per
    step, replayed as CUDA graphs from the fifth step on) and against maxUtts = 8 without graphs; six steps, reg > 0."""
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    p_g, v_g, c_g, opt_g = _train(8, 8, lens, nlabs, 6, useGraphs=True)
    p_e, v_e, c_e, _ = _train(8, 8, lens, nlabs, 6, useGraphs=False)
    p_a, v_a, c_a, opt_a = _train(3, 8, lens, nlabs, 6, useGraphs=True)
    assert len(opt_g._graphs) >= 1 and len(opt_a._graphs) == 0
    errs = dict(params_vs_graph=_rel(p_a, p_g), velocity_vs_graph=_rel(v_a, v_g), params_vs_eager=_rel(p_a, p_e),
                velocity_vs_eager=_rel(v_a, v_e), cost_rel_err_max=float(np.max(np.abs(c_a - c_g) / np.abs(c_g))))
    print(json.dumps({"sgd_accumulated_b8_m3": errs}))
    assert np.array_equal(p_g, p_e) and np.array_equal(v_g, v_e)      # graph replay = eager
    assert len(c_a) == len(c_g) == 6
    assert max(errs[k] for k in ("params_vs_graph", "velocity_vs_graph", "params_vs_eager", "velocity_vs_eager")) <= 1e-5
    assert errs["cost_rel_err_max"] <= 1e-5


def test_five_micro_batch_steps_do_not_overwrite_staging_buffers_in_use(cuda):
    """maxUtts = 2, batchSize = 10: five micro-batches per step cycle through the two staging buffers while the
    device is still reading them; every micro-batch must see its own utterances (the trajectory of one call per
    step shows it: a repacked buffer would change the gradient by far more than the tolerance)."""
    lens = [61, 23, 47, 35, 58, 19, 42, 30, 52, 27]
    nlabs = [12, 5, 9, 7, 14, 4, 8, 6, 11, 5]
    p_1, v_1, c_1, _ = _train(10, 10, lens, nlabs, 3)
    p_5, v_5, c_5, _ = _train(2, 10, lens, nlabs, 3)
    errs = dict(params=_rel(p_5, p_1), velocity=_rel(v_5, v_1), cost_rel_err_max=float(np.max(np.abs(c_5 - c_1) / np.abs(c_1))))
    print(json.dumps({"sgd_accumulated_b10_m2": errs}))
    assert errs["params"] <= 1e-5 and errs["velocity"] <= 1e-5 and errs["cost_rel_err_max"] <= 1e-5


# ------------------------------------------------------------------------------------------ 5. data parallel
WORKER = r'''
import os, sys
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tests")]
import numpy as np, torch, torch.distributed as dist
rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
if world > 1:
    dist.init_process_group("nccl")
import random, recipes, nnets.brnnet as rnnet, sgd
lens = [25, 30, 18, 30, 22, 27, 16, 29, 24, 19, 28, 21]
datas, labelss = recipes.synth_batch(13, 11, lens, [6, 8, 4, 9, 5, 7, 3, 8, 6, 4, 7, 5], seed=9)
keys = ["k%%d" %% i for i in range(len(lens))]
dd = dict(zip(keys, datas)); alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
np.random.seed(2); random.seed(33)
nn = rnnet.NNet(13, 11, 64, 3, 30, temporalLayer=2, reg=1e-3, maxUtts=2, maxLabels=10)
nn.initParams()
opt = sgd.SGD(nn, 30, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=7, verbose=False)
for _ in range(2):
    opt.run(dd, alis, list(keys), None)     # two steps per pass: 7 and 5 utterances
torch.cuda.synchronize()
np.save(os.path.join(sys.argv[1], "params_w%%d_r%%d.npy" %% (world, rank)), nn.params.cpu().numpy())
np.save(os.path.join(sys.argv[1], "cost_w%%d_r%%d.npy" %% (world, rank)), np.array(opt.costt))
if world > 1:
    dist.barrier(); dist.destroy_process_group()
'''


def test_two_rank_accumulated_steps_match_single_gpu(cuda, tmp_path):
    """batchSize = 7, maxUtts = 2, two ranks: the 7-utterance steps run 2 + 2 micro-batches, the 5-utterance ones
    2 + 1; temporalLayer = 2 and reg > 0, so both exchange buckets carry data.  Replicas bit-identical, and within
    1e-5 of one GPU accumulating the whole step (4 and 3 micro-batches)."""
    if cuda.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    p1_ = subprocess.Popen([sys.executable, str(script), str(tmp_path)], env=env, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
    p2_ = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", "29623", str(script), str(tmp_path)],
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
    print(json.dumps({"dp2_accumulated": dict(params_rel_err=err)}))
    assert np.array_equal(p20, p21)
    assert err < 1e-5
    c1, c2 = np.load(tmp_path / "cost_w1_r0.npy"), np.load(tmp_path / "cost_w2_r0.npy")
    np.testing.assert_allclose(c1, c2, rtol=1e-5)
