"""GPU tests of frame subsampling (ctcb_brnn_config.subsample = k at map subsampleLayer = L) on one H100.

1. The kernels alone (ctcb_frame_stack_f32 / ctcb_frame_unstack_f32) are exact copies: bit for bit against NumPy for
   k = 2, 3, 4, n odd and n % 4 == 0 (16-byte and, misaligned, 4-byte accesses), B = 1 and larger, Tmax < k and every
   T_u mod k; padding is zero and every output element is written.
2. The whole net against tests/net_oracle.py (compared by tests/net_check.py) for L = 1, L at the lowest temporal layer,
   L inside a stack, L above the temporal block and L = numLayers + 1, bi- and uni-directional, DNN, LSTM, layer norm
   and dropout: cost, every activation (S through what = 6) and every gradient tensor against the oracle's
   back-propagation through the GPU's own activations, with the bounds of tests/test_layernorm_gpu.py (relative, 1e-4).
3. Consistency: micro-batches and two emulated shards, graph replay, forward-only probabilities, the likelihood arks,
   runNNet end to end, checkpoints of the other width, check_grad on W_L, and the skip of utterances too short for
   their labels at the reduced rate.
Each comparison prints its measured errors as one JSON line (pytest -s)."""
import ctypes
import io
import json
import os
import struct

import numpy as np
import pytest

import recipes
from net_check import bits as _bits, compare, rel as _rel
from net_oracle import Net, frames

pytestmark = pytest.mark.gpu
FWD_TOL, GRAD_TOL = 1e-4, 1e-4


# ------------------------------------------------------------------------------------------------ 1. the kernels
def _np_stack(x, lens, k):
    Tmax, B, n = x.shape
    Tp = frames(Tmax, k)
    S = np.zeros((Tp, B, k * n), np.float32)
    for tp in range(Tp):
        for m in range(k):
            t = k * tp + m
            for u in range(B):
                if t < min(lens[u], Tmax):
                    S[tp, u, m * n:(m + 1) * n] = x[t, u]
    return S


def _np_unstack(dS, lens, k, Tmax):
    Tp, B, kn = dS.shape
    n = kn // k
    D = np.zeros((Tmax, B, n), np.float32)
    for t in range(Tmax):
        for u in range(B):
            if t < lens[u]:
                D[t, u] = dS[t // k, u, (t % k) * n:(t % k + 1) * n]
    return D


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("n,B,Tmax,misalign", [(13, 1, 9, 0), (13, 7, 17, 0), (64, 5, 23, 0), (64, 5, 23, 1),
                                              (8, 3, 1, 0), (12, 4, 3, 0), (1024, 9, 14, 0)])
def test_stack_and_unstack_are_exact_copies(k, n, B, Tmax, misalign, cuda):
    import _ctcb
    from _ctcb import lib, check, ptr
    rng = np.random.RandomState(k * 1000 + n + B)
    lens = [Tmax] + [int(x) for x in rng.randint(0, Tmax + 1, size=B - 1)]
    if B >= k + 1:                                  # every T_u mod k
        lens[1:k + 1] = [max(0, Tmax - r) for r in range(k)]
    Tp = frames(Tmax, k)
    x = rng.randn(Tmax, B, n).astype(np.float32)
    x[0, 0, 0] = -0.0
    dS = rng.randn(Tp, B, k * n).astype(np.float32)
    o = misalign                                    # a float's offset: 4-byte accesses on an n % 4 == 0 row
    d_x = cuda.from_numpy(np.concatenate([np.zeros(o, np.float32), x.ravel()])).cuda()[o:]
    d_ds = cuda.from_numpy(np.concatenate([np.zeros(o, np.float32), dS.ravel()])).cuda()[o:]
    d_lens = cuda.tensor(lens, dtype=cuda.int32).cuda()
    s_out = cuda.full((Tp * B * k * n + o,), float("nan"), device="cuda")[o:]
    d_out = cuda.full((Tmax * B * n + o,), float("nan"), device="cuda")[o:]
    t_out = cuda.full((B,), -1, dtype=cuda.int32, device="cuda")
    st = _ctcb.current_stream()
    check(lib.ctcb_frame_stack_f32(ptr(d_x), ptr(d_lens), Tmax, B, n, k, ptr(s_out), ptr(t_out), st))
    check(lib.ctcb_frame_unstack_f32(ptr(d_ds), ptr(d_lens), Tmax, B, n, k, ptr(d_out), st))
    S = s_out.cpu().numpy().reshape(Tp, B, k * n)
    D = d_out.cpu().numpy().reshape(Tmax, B, n)
    assert np.array_equal(S.view(np.uint32), _np_stack(x, lens, k).view(np.uint32))
    assert np.array_equal(D.view(np.uint32), _np_unstack(dS, lens, k, Tmax).view(np.uint32))
    assert t_out.cpu().numpy().tolist() == [frames(t, k) for t in lens]


# ------------------------------------------------------------------------------------------------ 2. the whole net
D_IN, K = 23, 17
# N, tl, nt, k, L, extra
NETS = {
    "bi_L1_k2": dict(H=64, N=3, tl=2, nt=1, k=2, sl=1, T=31, B=6, L=6),
    "bi_Ltl_k3": dict(H=64, N=3, tl=2, nt=1, k=3, sl=2, T=32, B=5, L=5),
    "uni_stack_inside_k2_h70": dict(H=70, N=4, tl=2, nt=2, k=2, sl=3, T=27, B=5, L=5, uni=True),
    "bi_above_k2_ln_dropout": dict(H=64, N=3, tl=1, nt=1, k=2, sl=3, T=29, B=6, L=6, ln=True, p=0.1),
    "bi_top_k3": dict(H=64, N=3, tl=2, nt=1, k=3, sl=4, T=31, B=5, L=5),
    "dnn_k2_ln": dict(H=64, N=3, tl=0, nt=0, k=2, sl=2, T=25, B=5, L=6, ln=True),
    "lstm_bi_Ltl_k2": dict(H=64, N=3, tl=2, nt=1, k=2, sl=2, T=26, B=5, L=6, cell="lstm"),
    "lstm_uni_L1_k3_ln": dict(H=64, N=3, tl=2, nt=1, k=3, sl=1, T=31, B=5, L=5, cell="lstm", uni=True, ln=True),
    "bi_Ltl_k2_h512": dict(H=512, N=3, tl=2, nt=1, k=2, sl=2, T=13, B=4, L=3),
}


def _kwargs(c, reg=0.0):
    """The keyword arguments of nnets.brnnet.NNet and net_oracle.Net that make net c."""
    return dict(temporalLayer=c["tl"] or -1, numTemporal=max(1, c["nt"]), reg=reg, unidirectional=bool(c.get("uni")),
                cell=c.get("cell", "relu"), dropout=c.get("p", 0.0), layerNorm=bool(c.get("ln")), subsample=c["k"],
                subsampleLayer=c["sl"])


def _gpu_net(c, B, reg=0.0, train=True):
    import nnets.brnnet as brnnet
    return brnnet.NNet(D_IN, K, c["H"], c["N"], c["T"], maxUtts=B, maxLabels=c["L"], train=train, **_kwargs(c, reg))


def _ragged(c, seed=5):
    """Lengths with every remainder mod k; label counts that fit ceil(T / k) frames."""
    T, B, L, k = c["T"], c["B"], c["L"], c["k"]
    rng = np.random.RandomState(seed)
    lens = [T] + [max(k, T - 1 - int(x)) for x in rng.randint(0, T // 2, size=B - 1)]
    lens[1:k] = [T - r for r in range(1, k)][:B - 1]
    nlabs = [int(rng.randint(1, max(1, min(L, frames(t, k) // 2)) + 1)) for t in lens]
    return lens, recipes.synth_batch(D_IN, K, lens, nlabs, seed=33)


@pytest.mark.parametrize("name", list(NETS))
def test_subsampled_net_matches_float64_oracle(name, cuda):
    c = NETS[name]
    lens, (datas, labelss) = _ragged(c)
    B, k, sl = c["B"], c["k"], c["sl"]
    reg = 1e-3
    np.random.seed(21)
    nn = _gpu_net(c, B, reg=reg)
    nn.initParams()
    np.random.seed(21)
    on = Net(D_IN, K, c["H"], c["N"], c["T"], **_kwargs(c, reg))
    on.initParams()
    for (w, b), (ow, ob) in zip(nn.stack, on.stack):        # the same draws, shapes (W_L k n wide) and order
        assert np.array_equal(w.cpu().numpy(), ow.astype(np.float32))
        assert np.array_equal(b.cpu().numpy(), ob.astype(np.float32))
    assert tuple(nn.stack[sl - 1][0].shape)[1] == k * (D_IN if sl == 1 else c["H"])
    nn.costAndGradBatch(datas, labelss)
    r = compare(nn, on, datas, labelss, lens)
    assert np.array_equal(r["skips"], r["skips_own"]) and not r["skips"].any()
    for u in range(B):                                      # S is zero beyond T'_u
        assert not np.any(r["acts"][6, 0][frames(lens[u], k):, u])
    cost_err, fwd = r["cost_own"], max(r["fwd"]["X"] + [r["fwd"]["S"]])
    grad_err, grad_elem, plain = r["grad_given"], r["grad_given_elem"], r["grad_plain"]
    print(json.dumps({"subsample_net_" + name: dict(cost=cost_err, fwd=fwd, grad_given_frob_max=max(grad_err),
                                                    grad_given_elem_max=max(grad_elem), grad_plain_frob_max=max(plain))}))
    assert cost_err <= FWD_TOL and fwd <= FWD_TOL
    assert max(grad_err) <= GRAD_TOL, grad_err


# ------------------------------------------------------------------------------------------------ 3. consistency
def _small(maxUtts, reg=0.0, uni=False, dropout=0.0, k=2, sl=2, train=True):
    import nnets.brnnet
    np.random.seed(4)
    nn = nnets.brnnet.NNet(13, 11, 64, 4, 60, temporalLayer=2, reg=reg, maxUtts=maxUtts, maxLabels=20,
                           unidirectional=uni, dropout=dropout, subsample=k, subsampleLayer=sl, train=train)
    nn.initParams()
    return nn


def _batch8(seed=7):
    lens = [50, 37, 12, 45, 29, 60, 21, 40]
    nlabs = [9, 14, 5, 11, 5, 20, 3, 7]
    return recipes.synth_batch(13, 11, lens, nlabs, seed=seed)


@pytest.mark.parametrize("uni,dropout,sl", [(False, 0.0, 2), (True, 0.1, 3), (False, 0.1, 1)])
def test_micro_batches_and_two_shards_match_one_call(uni, dropout, sl, cuda):
    import _ctcb
    import parallel
    from _ctcb import lib, check, ptr
    reg = 1e-2
    datas, labelss = _batch8()
    full = _small(8, reg, uni, dropout, sl=sl)
    c1, _, _ = full.costAndGradBatch(datas, labelss)
    g1 = full.grads_ext[:full.nparams + 4].cpu().numpy().astype(np.float64)
    split = _small(3, reg, uni, dropout, sl=sl)     # three micro-batches of 3, 3, 2
    c2, _, _ = split.costAndGradBatch(datas, labelss)
    g2 = split.grads_ext[:split.nparams + 4].cpu().numpy().astype(np.float64)
    total, last = None, None
    for rank in range(2):
        idx = parallel.shard(list(range(8)), rank, 2)
        nn = _small(4, reg, uni, dropout, sl=sl)
        nn.dropoutShard = (rank, 2)
        check(lib.ctcb_brnn_set_deferred_l2(nn._h, 1))
        nn.costAndGradBatch([datas[i] for i in idx], [labelss[i] for i in idx])
        part = nn.grads_ext[:nn.nparams + 4].clone()
        total = part if total is None else total + part
        last = nn
    check(lib.ctcb_brnn_apply_l2_f32(last._h, ptr(last.params), ptr(total), _ctcb.current_stream()))
    g3 = total.cpu().numpy().astype(np.float64)
    e_micro, e_shard = _rel(g2[:-4], g1[:-4]), _rel(g3[:-4], g1[:-4])
    print(json.dumps({"subsample_accum_%s_p%g_L%d" % ("uni" if uni else "bi", dropout, sl):
                      dict(micro=e_micro, shards=e_shard, cost=float(np.max(np.abs(c2 - c1))))}))
    assert np.allclose(c1, c2, rtol=1e-6)
    assert e_micro < 1e-5 and e_shard < 1e-5
    assert g2[-4] == g3[-4] == g1[-4] == 8 and g1[-1] == g2[-1] == g3[-1] == 0


def _train(useGraphs, optimizer="nesterov", dropout=0.0, steps=5, uni=False, alpha=1e-3):
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
    opt = sgd.SGD(nn, 60, alpha=alpha, momentum=0.9, maxGradNorm=5.0, batchSize=8, verbose=False, optimizer=optimizer)
    opt.useGraphs = useGraphs
    for _ in range(steps):
        opt.run(dd, alis, list(keys), None)
    torch.cuda.synchronize()
    return nn.params.cpu().numpy(), np.array(opt.costt), opt


@pytest.mark.parametrize("optimizer,dropout,uni", [("nesterov", 0.0, False), ("adam", 0.1, True),
                                                   ("nesterov", 0.1, False), ("adam", 0.0, False)])
def test_graph_replay_is_bit_identical_to_eager_steps(optimizer, dropout, uni, cuda):
    p_g, c_g, opt_g = _train(True, optimizer, dropout, uni=uni)
    p_e, c_e, opt_e = _train(False, optimizer, dropout, uni=uni)
    print(json.dumps({"subsample_graph_%s_p%g_%s" % (optimizer, dropout, "uni" if uni else "bi"):
                      dict(graphs=len(opt_g._graphs), costs=c_g.tolist())}))
    assert len(opt_g._graphs) >= 1 and len(opt_e._graphs) == 0
    assert np.array_equal(p_g, p_e) and np.array_equal(c_g, c_e)
    assert np.isfinite(p_g).all()


def test_training_lowers_the_cost(cuda):
    _, costs, _ = _train(True, "adam", steps=20, alpha=1e-3)
    print(json.dumps({"subsample_adam_costs": costs.tolist()}))
    assert np.isfinite(costs).all() and costs[-1] < 0.9 * costs[0]


def test_forward_only_probs_are_bit_identical_to_a_training_call(cuda):
    for name in ("bi_L1_k2", "uni_stack_inside_k2_h70", "dnn_k2_ln", "lstm_bi_Ltl_k2", "bi_top_k3", "lstm_uni_L1_k3_ln"):
        c = NETS[name]
        lens, (datas, labelss) = _ragged(c)
        np.random.seed(3)
        nn = _gpu_net(dict(c, p=0.0), c["B"])
        nn.initParams()
        batch = nn._batch.pack(datas, labelss).upload()
        Tp = frames(batch.Tmax, c["k"])
        nn.costAndGradDevice(batch, want_probs=True)
        p_train = _bits(nn._probs_view(batch.B, Tp).clone())
        p_fwd = _bits(nn._forward_device(batch).clone())
        assert p_fwd.size == Tp * batch.B * K
        assert np.array_equal(p_train, p_fwd), name
        np.random.seed(3)
        inf = _gpu_net(dict(c, p=0.0), c["B"], train=False)
        inf.initParams()
        out = inf.forwardBatch(datas)
        probs = p_fwd.view(np.float32).reshape(Tp, batch.B, K)
        for u, d in enumerate(datas):
            assert out[u].shape == (K, frames(d.shape[1], c["k"]))
            assert np.array_equal(out[u], probs[:frames(d.shape[1], c["k"]), u, :].T), name
        assert inf.costAndGrad(datas[1]).shape == out[1].shape


def test_forward_batch_on_a_training_net_with_lstm_layers_from_map_1(cuda):
    """C2 with LSTM layers at k = 2 from map 1: a training net's forward-only calls (forwardBatch) run in its training
    workspace and give the probabilities of a training call, bit for bit."""
    import nnets.brnnet as brnnet
    np.random.seed(5)
    nn = brnnet.NNet(41, 62, 512, 2, 200, temporalLayer=1, maxUtts=32, maxLabels=30, cell="lstm", subsample=2,
                     subsampleLayer=1)
    nn.initParams()
    from _ctcb import lib
    assert nn.train and nn._ws.numel() == lib.ctcb_brnn_workspace_bytes(ctypes.byref(nn._cfg))
    lens = [200, 199, 150, 77, 31, 2]
    datas, labelss = recipes.synth_batch(41, 62, lens, [20, 20, 15, 9, 3, 1], seed=6)
    batch = nn._batch.pack(datas, labelss).upload()
    nn.costAndGradDevice(batch, want_probs=True)
    p_train = _bits(nn._probs_view(batch.B, 100).clone()).view(np.float32).reshape(100, len(lens), 62)
    out = nn.forwardBatch(datas)
    for u, T in enumerate(lens):
        assert out[u].shape == (62, frames(T, 2))
    # forwardBatch sorts its micro-batch by length; the forward-only call of the training call's batch is compared bits
    p_fwd = _bits(nn._forward_device(batch).clone()).view(np.float32).reshape(100, len(lens), 62)
    assert np.array_equal(p_train.view(np.uint32), p_fwd.view(np.uint32))
    for u, T in enumerate(lens):       # the same utterances in another order of the batch
        assert np.allclose(out[u], p_fwd[:frames(T, 2), u, :].T, rtol=1e-5, atol=1e-7)


def test_short_utterances_are_skipped(cuda):
    """ceil(T / k) below what the labels need: 7 frames at k = 3 give 3, too few for 3 labels with a repeat (the CTC
    skips it; the others of the batch train as usual) or for 4 labels (the host rule drops it before a step)."""
    import parallel
    nn = _small(4, k=3, sl=1)
    datas, _ = recipes.synth_batch(13, 11, [7, 7, 7, 30], [1, 1, 1, 1], seed=2)
    labelss = [np.array([1, 2, 3, 4], np.int32), np.array([1, 2, 2], np.int32), np.array([1, 2, 3], np.int32),
               np.array([3, 4, 5], np.int32)]
    costs, _, skips = nn.costAndGradBatch(datas[1:], labelss[1:])
    assert skips.tolist() == [True, False, False], skips
    assert np.isfinite(costs[1:]).all()
    dd = {"a": datas[0], "b": datas[1], "c": datas[2], "d": datas[3]}
    alis = {"a": labelss[0], "b": labelss[1], "c": labelss[2], "d": labelss[3]}
    assert parallel.select_step_utterances(dd, alis, list("abcd"), 60, 0, 1, subsample=3) == list("bcd")


def test_write_log_likes_writes_the_reduced_frames(cuda, tmp_path):
    import writeLikelihoods
    nn = _small(4, k=3, sl=2, train=False)
    lens = [10, 31, 8, 20, 9]
    datas, _ = recipes.synth_batch(13, 11, lens, [1] * 5, seed=4)

    class Loader(object):
        def loadDataFileDict(self, fn):
            keys = ["u%d" % i for i in range(len(lens))]
            return dict(zip(keys, datas)), None, keys, np.array(lens)
    lik = writeLikelihoods.writeLogLikes(Loader(), nn, 1, str(tmp_path))
    raw = open(str(tmp_path / "loglikelihoods1.ark"), "rb").read()
    pos = 0
    for i, T in enumerate(lens):
        key = ("u%d " % i).encode()
        assert raw[pos:pos + len(key)] == key
        pos += len(key) + 1 + 4 + 1
        rows = struct.unpack("i", raw[pos:pos + 4])[0]
        pos += 4 + 1
        cols = struct.unpack("i", raw[pos:pos + 4])[0]
        pos += 4
        assert (rows, cols) == (frames(T, 3), 11)
        body = np.frombuffer(raw[pos:pos + 4 * rows * cols], np.float32).reshape(rows, cols)
        assert np.array_equal(body, lik["u%d" % i].T)
        pos += 4 * rows * cols
    assert pos == len(raw)


def test_checkpoints_round_trip_and_refuse_the_other_width(cuda):
    import sgd
    a = _small(8)
    f = io.BytesIO()
    a.toFile(f)
    f.seek(0)
    b = _small(8)
    b.fromFile(f)
    assert np.array_equal(a.params.cpu().numpy(), b.params.cpu().numpy())
    for other in (_small(8, k=1), _small(8, k=3)):
        f = io.BytesIO()
        other.toFile(f)
        f.seek(0)
        with pytest.raises(ValueError, match="subsampl"):
            b.fromFile(f)
        f = io.BytesIO()
        sgd.SGD(other, 60, verbose=False).toFile(f)
        f.seek(0)
        with pytest.raises(ValueError, match="subsampl"):
            sgd.SGD(b, 60, verbose=False).fromFile(f)
    f = io.BytesIO()
    _small(8, k=1).toFile(f)
    f.seek(0)
    with pytest.raises(ValueError) as e:
        b.fromFile(f)
    assert "(64, 64)" in str(e.value) and "(64, 128)" in str(e.value)


def test_run_nnet_trains_resumes_and_tests_a_subsampled_net(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    from run_utils import dump_config, load_config
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=9, rawsize=20, outputDim=9, T_range=(12, 39), L_range=(2, 5))
    args = ["--layerSize", "64", "--numLayers", "3", "--temporalLayer", "2", "--subsample", "2", "--subsampleLayer",
            "2", "--epochs", "1", "--step", "1e-3", "--dataDir", data, "--numFiles", "2", "--inputDim", "16",
            "--rawDim", "20", "--outputDim", "9", "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4",
            "--save_every", "1", "--runDir", str(tmp_path / "runs"), "--quiet"]
    _, net = runNNet.run(args)
    assert (net.subsample, net.subsampleLayer) == (2, 2) and tuple(net.stack[1][0].shape) == (64, 128)
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg_file = os.path.join(run_dir, "cfg.json")
    cfg = load_config(cfg_file)
    assert (cfg["subsample"], cfg["subsampleLayer"]) == (2, 2)
    p_epoch0 = net.params.cpu().numpy().copy()
    cfg["epochs"] = 2
    dump_config(cfg, cfg_file)
    _, net2 = runNNet.run(["--cfg_file", cfg_file, "--quiet"])
    assert net2.subsample == 2 and np.array_equal(p_epoch0, net2.params.cpu().numpy())
    out = str(tmp_path / "arks")
    tnet = runNNet.run(["--cfg_file", cfg_file, "--test", "--dataDir", data, "--numFiles", "2", "--outDir", out,
                        "--maxUtts", "4"])
    assert tnet.subsample == 2 and not tnet.train
    assert np.array_equal(tnet.params.cpu().numpy(), p_epoch0)
    loader = dl.DataLoader(data, 20, 16, data)
    _, _, keys, sizes = loader.loadDataFileDict(1)
    raw = open(os.path.join(out, "loglikelihoods1.ark"), "rb").read()
    key = (keys[0] + " ").encode()
    assert raw.startswith(key)
    assert struct.unpack("i", raw[len(key) + 6:len(key) + 10])[0] == frames(int(sizes[0]), 2)


def test_check_grad_on_w_l(cuda):
    """NNet.check_grad (forward differences in fp32, as test_brnn_gpu.py) on every matrix, W_L = 8 x 12 included, with
    one utterance whose length is not a multiple of k."""
    import nnets.brnnet as rnnet
    datas, labelss = recipes.synth_batch(6, 5, [13], [3], seed=4)
    np.random.seed(8)
    nn = rnnet.NNet(6, 5, 8, 2, 13, temporalLayer=1, subsample=2, subsampleLayer=1)
    nn.initParams()
    assert tuple(nn.stack[0][0].shape) == (8, 12)
    pairs = nn.check_grad(datas[0], labelss[0], epsilon=1e-3, maxChecks=12, verbose=False)
    ana = np.array([p[0] for p in pairs])
    num = np.array([p[1] for p in pairs])
    w_l = slice(0, 8 * 12)
    print(json.dumps({"subsample_check_grad": dict(max_err=float(np.abs(ana - num).max()),
                                                   w_l_max_err=float(np.abs(ana[w_l] - num[w_l]).max()))}))
    assert np.abs(ana - num).max() < 0.05 * max(1.0, np.abs(ana).max())
