"""GPU tests of whole nets in TF32 mode (NNet(..., tf32=True), ctcb_brnn_config.tf32 = 1) on one H100.

Stages from their own inputs: after one training call, read through ctcb_brnn_activation_offset (the hooks of
test_step_reductions_gpu.py), every weight gradient dW_j = delta_j^T X_{j-1} and every plainly stored forward map
(X_j = ReLU(X_{j-1} W_j^T + b_j) of a feed-forward layer, the logits) is checked against float64 of the call's own
float32 operands at the plan ctcb_debug_gemm_plan_tf32 reports for the call's own pointers: on the tensor cores with the
operands rounded by rna and the rounded-operand bound of test_gemm_tf32_gpu.py, on the FFMA kernel with the operands as
they are and its bound in test_gemm_plans_gpu.py.  The tensor-core ReLU sweep's forward states are checked step-locally
from the call's own states and pre-activations (test_sweep_tf32_gpu.py; a bi-directional layer's pre-activation is
recomputed with ctcb_gemm_tf32 at the call's plan, which is deterministic).  Negative controls: float64 of the unrounded
operands (a stage that ran fp32-faithful) misses each tensor-core stage with K <= CONTROL_MAX_K, and the truncation
emulation each sweep, by at least MARGIN bounds.  With every contraction on the FFMA kernel (CTCB_GEMM=simt) and the
cluster sweep, a TF32 net computes the mode-off net's bytes.
Consistency: workspace sizes are those of the mode-off net; micro-batches and two emulated shards agree with one call;
graph replay is bit for bit with eager steps; forwardBatch gives the training call's probabilities bit for bit.
Learning: a few hundred steps on a synthetic task whose labels are a function of the features bring the cost down as
the fp32-faithful run from the same start does.  runNNet trains, resumes and runs --test with --tf32, and checkpoints
load across the modes.  Each test prints its numbers as one JSON line (pytest -s)."""
import json
import os

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, rel as _rel
from recipes import knobs  # noqa: F401  (fixture)
from test_gemm_plans_gpu import BOUNDS as GEMM_BOUNDS, FIELDS as GEMM_FIELDS, _chain as gemm_chain
from test_gemm_tf32_gpu import CONTROL_MAX_K, MARGIN, TF32_BOUND, _rna_t
from test_step_reductions_gpu import D_IN, MAXB, MAXT, _batches, _hook, _map_input, _ws_array
from test_sweep_tf32_gpu import TF32_C0, TF32_C1, _steps_tf32

pytestmark = pytest.mark.gpu
U = 2.0 ** -24

NETS = {
    "bi_relu_h1024": dict(H=1024, N=2, K=30, kw=dict(temporalLayer=1)),
    "uni_relu_h1024": dict(H=1024, N=3, K=30, kw=dict(temporalLayer=2, unidirectional=True)),
    "lstm_uni_h1024": dict(H=1024, N=2, K=30, kw=dict(temporalLayer=1, cell="lstm", unidirectional=True)),
    "sub_inter_cond_ln_h256": dict(H=256, N=4, K=37, kw=dict(temporalLayer=3, layerNorm=True, subsample=2,
                                                             subsampleLayer=2, interLayer=2, interWeight=0.3,
                                                             selfCondition=True)),
}


def _net(c, tf32=True):
    import nnets.brnnet as brnnet
    np.random.seed(17)
    nn = brnnet.NNet(D_IN, c["K"], c["H"], c["N"], MAXT, maxUtts=MAXB, maxLabels=6, tf32=tf32, **c["kw"])
    nn.initParams()
    rng = np.random.RandomState(2)
    for w, b in nn.stack[:c["N"] + 1]:
        b.copy_(nn._torch.from_numpy((0.1 * rng.randn(*b.shape)).astype(np.float32)))
    if nn.selfCondition:
        nn.stack[-1][0].copy_(nn._torch.from_numpy(rng.uniform(-0.4, 0.4, tuple(nn.stack[-1][0].shape))
                                                   .astype(np.float32)))
    return nn


def _plan(ta, tb, M, N, K, a, lda, b, ldb):
    import ctypes
    from _ctcb import lib, check
    out = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_gemm_plan_tf32(ta, tb, M, N, K, a, lda, b, ldb, 1, out))
    return dict(zip(GEMM_FIELDS, list(out)))


def _ref(plan, A, B, K):
    """(float64 A B, |A| |B|, bound coefficient, float64 A B of the unrounded operands or None) as the plan's kernel
    computes it: rounded operands on the tensor cores, the operands themselves on the FFMA kernel.  A, B: device
    float32.  The last one is the negative control of a tensor-core stage."""
    plain = None
    if plan["kernel"] == 1:
        plain = (A.double() @ B.double()).cpu().numpy()
        A, B = _rna_t(A), _rna_t(B)
        c0, c1 = TF32_BOUND
    else:
        c0, c1 = GEMM_BOUNDS[0]
    a, b = A.double(), B.double()
    return ((a @ b).cpu().numpy(), (a.abs() @ b.abs()).cpu().numpy(), c0 + c1 * gemm_chain(plan, K), plain)


def _control(plan, K, got, plain, S, coef):
    """The unrounded operands' miss in bounds, where the stage ran on the tensor cores and K <= CONTROL_MAX_K."""
    if plain is None or K > CONTROL_MAX_K:
        return None
    return _ratio(np.abs(got - plain), S, coef)


def _ratio(err, S, coef):
    lim = coef * U * S
    r = np.where(lim > 0, err / np.maximum(lim, 1e-300), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def _temporal(nn, i):
    return nn.numTemporal and nn.temporalLayer <= i < nn.temporalLayer + nn.numTemporal


def _frames(nn, batch, j):
    return nn.frames(batch.Tmax) if nn.subsample > 1 and j >= nn.subsampleLayer else batch.Tmax


def _weight(nn, j):
    w = nn.stack[j - 1][0]
    return w, w.data_ptr()


def _input(nn, batch, j):
    """(device [T][B][cols], pointer) of what map j read: X'_m above the conditioned layer, else _map_input's."""
    if nn.selfCondition and j - 1 == nn.interLayer:
        T = _frames(nn, batch, j - 1)
        off, w = _hook(nn, 12, 0)
        x = _ws_array(nn, off, T, batch.B, w)
        return x, x.data_ptr()
    return _map_input(nn, j, batch)


def _dW(nn, batch, j, grads):
    """Ratio of dW_j to the reference of its plan, from the call's delta and the input the map read."""
    T, B = _frames(nn, batch, j), batch.B
    off, rows = _hook(nn, 7, j)
    dd = _ws_array(nn, off, T, B, rows).reshape(T * B, rows)
    x, xp = _input(nn, batch, j)
    cols = x.shape[2]
    x = x.reshape(T * B, cols)
    plan = _plan(1, 0, rows, cols, T * B, dd.data_ptr(), rows, xp, cols)
    P, S, coef, plain = _ref(plan, dd.T, x, T * B)
    wv = nn.grad[j - 1][0]
    o = (wv.data_ptr() - nn.grads.data_ptr()) // 4
    got = grads[o:o + rows * cols].reshape(rows, cols).astype(np.float64)
    return plan["kernel"], _ratio(np.abs(got - P), S, coef), _control(plan, T * B, got, plain, S, coef)


def _fwd(nn, batch, j):
    """Ratio of the stored output of map j (a feed-forward ReLU layer, or the logits) to the reference of its plan."""
    T, B = _frames(nn, batch, j), batch.B
    x, xp = _input(nn, batch, j)
    cols = x.shape[2]
    x = x.reshape(T * B, cols)
    W, Wp = _weight(nn, j)
    rows = W.shape[0]
    plan = _plan(0, 1, T * B, rows, cols, xp, cols, Wp, cols)
    P, S, coef, plain = _ref(plan, x, W.T, cols)
    b = nn.stack[j - 1][1].reshape(-1).double().cpu().numpy()
    relu = (lambda v: np.maximum(v, 0.0)) if j <= nn.numLayers else (lambda v: v)      # noqa: E731
    want, S = relu(P + b), S + np.abs(b)
    off, w = _hook(nn, 0, j)
    got = _ws_array(nn, off, T, B, w).reshape(T * B, w).double().cpu().numpy()
    return (plan["kernel"], _ratio(np.abs(got - want), S, coef),
            _control(plan, cols, got, None if plain is None else relu(plain + b), S, coef))


def _pre(nn, batch, i):
    """The pre-activation map i wrote for temporal layer i ([T][B][H] host): read where it survives (a uni-directional
    layer), else recomputed with ctcb_gemm_tf32 at the call's plan."""
    import _ctcb
    import torch
    from _ctcb import lib, check
    T, B, H = _frames(nn, batch, i), batch.B, nn.layerSize
    if nn.unidirectional:
        off, w = _hook(nn, 0, i)
        return _ws_array(nn, off, T, B, w).cpu().numpy()
    x, xp = _input(nn, batch, i)
    cols = x.shape[2]
    W, Wp = _weight(nn, i)
    out = torch.zeros(T * B * H, device="cuda")
    wsb = int(lib.ctcb_gemm_workspace_bytes(T * B, H, cols))
    ws = torch.zeros(max(wsb, 16), dtype=torch.uint8, device="cuda")
    check(lib.ctcb_gemm_tf32(0, 1, T * B, H, cols, 1.0, xp, cols, Wp, cols, 0.0, out.data_ptr(), H,
                             nn.stack[i - 1][1].data_ptr(), 0, None, ws.data_ptr(), wsb, _ctcb.current_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(T, B, H)


class _Sw:
    def __init__(self, T, lens, ndir):
        self.T, self.lens, self.ndir = T, np.asarray(lens), ndir


def _sweep_fwd(nn, batch, lens, i):
    """Step-local ratio of For (and Back) of ReLU temporal layer i to the TF32 sweep's bound, its truncation control."""
    T, B, H = _frames(nn, batch, i), batch.B, nn.layerSize
    ndir = 1 if nn.unidirectional else 2
    outs = [_ws_array(nn, _hook(nn, 1 + q, i)[0], T, B, H).cpu().numpy() for q in range(ndir)]
    base = nn.numLayers + 1 + (i - nn.temporalLayer) * ndir
    Ms = [nn.stack[base + d][0].cpu().numpy().T for d in range(ndir)]
    import ctypes
    from _ctcb import lib, check
    plan = (ctypes.c_int32 * 8)()
    check(lib.ctcb_debug_sweep_plan_tf32(H, B, ndir, plan))
    assert plan[0] == 2, list(plan)
    bound = TF32_C0 + TF32_C1 * (H // plan[2] // 32)
    w = _steps_tf32(_Sw(T, lens, ndir), outs, _pre(nn, batch, i), Ms, None, bound, outs)
    return w["ratio"] / bound, w["trunc"]


@pytest.mark.parametrize("name", list(NETS))
def test_stages_from_their_own_inputs(name, cuda):
    torch = cuda
    c = NETS[name]
    nn = _net(c)
    lens, (datas, labelss) = _batches(c, 41)
    batch = nn.swap_batches().pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, want_probs=True)
    torch.cuda.synchronize()
    grads = nn.grads.cpu().numpy()
    rep, kernels, neg = {}, set(), {}
    N = nn.numLayers
    for j in range(1, N + 2):
        if not (j == N + 1 and nn.interLayer):      # (dW_{N+1} also holds the intermediate head's term)
            k, rep["dW%d" % j], neg["dW%d" % j] = _dW(nn, batch, j, grads)
            kernels.add(k)
        plain = j == N + 1 or not (_temporal(nn, j) or nn.layerNorm or j == nn.interLayer and nn.selfCondition)
        if plain:
            k, rep["fwd%d" % j], neg["fwd%d" % j] = _fwd(nn, batch, j)
            kernels.add(k)
    for i in range(1, N + 1):
        if _temporal(nn, i) and nn.cell == "relu" and nn.layerSize >= 1024:
            rep["sweep%d" % i], neg["sweep%d" % i] = _sweep_fwd(nn, batch, lens, i)
    neg = {k: v for k, v in neg.items() if v is not None}
    print(json.dumps({"tf32_stages_" + name: dict(ratios=rep, kernels=sorted(kernels), negative_controls=neg)}))
    assert 1 in kernels and neg
    assert max(rep.values()) <= 1.0, rep
    assert min(neg.values()) >= MARGIN, neg


def test_ffma_stages_have_the_mode_off_bytes(knobs, cuda):
    """The FFMA contraction (CTCB_GEMM=simt), the cluster sweep (H = 64), the CTC, the column sums and the update
    have no TF32 mode: with every contraction on the FFMA kernel the whole call is the mode-off one, bit for bit."""
    knobs("CTCB_GEMM", "simt")
    c = dict(H=64, N=3, K=35, kw=dict(temporalLayer=2))
    lens, (datas, labelss) = _batches(c, 41)
    out = []
    for tf32 in (False, True):
        nn = _net(c, tf32=tf32)
        costs, _, _ = nn.costAndGradBatch(datas, labelss)
        out.append((costs, _bits(nn.grads_ext)))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


# ------------------------------------------------------------------------------------------------ consistency
def _small(maxUtts, tf32=True, H=1024):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, H, 3, 60, temporalLayer=2, reg=1e-2, maxUtts=maxUtts, maxLabels=20, tf32=tf32)
    nn.initParams()
    return nn


def _ragged(seed=7):
    lens = [50, 37, 12, 44, 29, 60, 21, 40]
    nlabs = [9, 14, 8, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


def test_workspaces_do_not_depend_on_the_mode(cuda):
    a, b = _small(8, False), _small(8, True)
    assert a._cfg.tf32 == 0 and b._cfg.tf32 == 1
    assert a._ws.numel() == b._ws.numel() and a.nparams == b.nparams
    import ctypes
    from _ctcb import lib
    for fn in (lib.ctcb_brnn_workspace_bytes, lib.ctcb_brnn_error_flag_offset):
        assert fn(ctypes.byref(a._cfg)) == fn(ctypes.byref(b._cfg))
    assert (lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(a._cfg), None)
            == lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(b._cfg), None))


def test_micro_batches_and_two_shards_match_one_call(cuda):
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    datas, labelss = _ragged()
    full = _small(8)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    g1 = full.grads_ext[:full.nparams + 4].cpu().numpy().astype(np.float64)
    split = _small(3)
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 4].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    print(json.dumps({"tf32_accum": dict(micro=e_micro, shards=e_shard)}))
    # The fp32-faithful tests hold this to 1e-5, the reordering of the sums.  In TF32 mode a last-bit difference of that
    # reordering can move an operand across a TF32 rounding boundary, a step of 2^-11 of that element: measured 1.7e-5
    # (micro-batches) and 7.4e-7 (shards) on an H100.
    assert np.allclose(c1, c2, rtol=1e-5)
    assert e_micro < 1e-4 and e_shard < 1e-4


def _train(useGraphs, steps=6):
    import random
    import sgd
    import torch
    lens, nlabs = [50, 37, 44, 29, 60, 21, 40, 33], [9, 14, 11, 5, 20, 3, 7, 8]
    datas, labelss = recipes.synth_batch(13, 11, lens, nlabs, seed=9)
    keys = ["k%d" % i for i in range(len(lens))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    nn = _small(8)
    random.seed(33)
    opt = sgd.SGD(nn, 60, alpha=1e-3, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn, np.array(opt.costt), opt


def test_graph_replay_is_bit_identical_to_eager_steps(cuda):
    nn_g, c_g, opt_g = _train(True)
    nn_e, c_e, opt_e = _train(False)
    print(json.dumps({"tf32_graph": dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1
    assert np.array_equal(nn_g.params.cpu().numpy(), nn_e.params.cpu().numpy()) and np.array_equal(c_g, c_e)


def test_forward_batch_has_the_training_call_probabilities(cuda):
    import torch
    datas, labelss = _ragged()
    nn = _small(8)
    batch = nn.swap_batches().pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, want_probs=True)
    p_train = nn._probs_view(batch.B, batch.Tmax).cpu().numpy()
    torch.cuda.synchronize()
    out = nn.forwardBatch(datas)
    for u, d in enumerate(datas):
        want = np.ascontiguousarray(p_train[:d.shape[1], u, :].T)
        assert np.array_equal(out[u].view(np.uint32), want.view(np.uint32)), u


# ------------------------------------------------------------------------------------------------ learning
def _task(n=64, T=30, D=13, K=6, seed=3):
    """Utterances whose labels are a function of the features: frame t belongs to class argmax of a fixed projection
    of its features, and the labels are the runs of that class sequence."""
    rng = np.random.RandomState(seed)
    P = rng.randn(D, K - 1)
    datas, labelss = [], []
    for _ in range(n):
        x = rng.randn(D, T).astype(np.float32)
        cls = np.argmax(P.T @ x, axis=0) + 1
        labs = [int(cls[0])] + [int(b) for a, b in zip(cls[:-1], cls[1:]) if a != b]
        datas.append(x)
        labelss.append(labs[:20])
    return datas, labelss


def _learn(tf32, steps):
    import random
    import nnets.brnnet
    import sgd
    datas, labelss = _task()
    keys = ["u%d" % i for i in range(len(datas))]
    dd = dict(zip(keys, datas))
    alis = dict(zip(keys, [list(map(str, l)) for l in labelss]))
    np.random.seed(12)
    nn = nnets.brnnet.NNet(13, 6, 1024, 2, 30, temporalLayer=1, maxUtts=16, maxLabels=20, tf32=tf32)
    nn.initParams()
    random.seed(33)
    opt = sgd.SGD(nn, 30, alpha=3e-4, optimizer="adam", batchSize=16, verbose=False)
    for _ in range(steps // (len(keys) // 16)):
        opt.run(dd, alis, list(keys), None)
    c = np.array(opt.costt)
    return float(c[:4].mean()), float(c[-4:].mean())


# The cost is the mean CTC loss per utterance.  Criterion: the TF32 run ends below a quarter of where it started, and
# within 20 % (plus 0.05) of where the fp32-faithful run from the same start ends.  The margin was set from the two
# runs of this test on an H100 (DESIGN.md section 6).
LEARN_STEPS, LEARN_DROP, LEARN_TOL = 320, 0.25, 0.2


def test_tf32_learns_as_the_fp32_faithful_run(cuda):
    s_off, e_off = _learn(False, LEARN_STEPS)
    s_on, e_on = _learn(True, LEARN_STEPS)
    print(json.dumps({"tf32_learning": dict(steps=LEARN_STEPS, fp32=[s_off, e_off], tf32=[s_on, e_on])}))
    assert s_on == pytest.approx(s_off, rel=1e-2)
    assert e_on <= LEARN_DROP * s_on
    assert e_on <= (1 + LEARN_TOL) * e_off + 0.05


# ------------------------------------------------------------------------------------------------ end to end
def test_run_nnet_trains_resumes_and_tests_with_tf32(cuda, tmp_path):
    import dataLoader as dl
    import nnets.brnnet
    import pickle
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    args = ["--layerSize", "1024", "--numLayers", "2", "--temporalLayer", "1", "--tf32", "--epochs", "1", "--step",
            "1e-4", "--dataDir", data, "--numFiles", "2", "--inputDim", "16", "--rawDim", "20", "--outputDim", "9",
            "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1", "--runDir",
            str(tmp_path / "runs"), "--quiet"]
    opt, net = runNNet.run(args)
    assert net.tf32 and net._cfg.tf32 == 1
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert cfg["tf32"] is True
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.tf32 and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert not tnet.train and tnet.tf32
    for fn in (1, 2):
        assert os.path.getsize(os.path.join(out, "loglikelihoods%d.ark" % fn)) > 9 * 16
    # the checkpoint loads into a net of either mode (no parameter depends on it); their probabilities agree to the
    # TF32 rounding
    probs = []
    datas = [np.random.RandomState(5).randn(16, 30).astype(np.float32)]
    for tf32 in (False, True):
        nn = nnets.brnnet.NNet(16, 9, 1024, 2, 40, temporalLayer=1, train=False, tf32=tf32)
        nn.initParams()
        with open(os.path.join(run_dir, "params.pk"), "rb") as fid:
            pickle.load(fid)
            nn.fromFile(fid)
        probs.append((nn.params.cpu().numpy(), nn.forwardBatch(datas)[0]))
    assert np.array_equal(probs[0][0], probs[1][0])
    probs = [p for _, p in probs]
    assert np.abs(probs[0] - probs[1]).max() < 1e-2
