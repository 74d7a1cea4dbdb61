"""GPU tests of batched inference: forward-only calls in the forward workspace layout (ctcb_brnn_forward_workspace_bytes)
give the same bits as a training call, NNet.forwardBatch matches the float64 oracle utterance by utterance, and the
likelihood writer (writeLikelihoods.writeLogLikes, runNNet --test --maxUtts) writes the arks the per-utterance loop
writes."""
import ctypes
import json
import os
import pickle
import struct

import numpy as np
import pytest

import recipes
from oracle import brnn_oracle

pytestmark = pytest.mark.gpu

# name: (H, N, temporal layer, unidirectional, utterance lengths, expected sweep kernel: 1 cluster / 2 tensor core
#        [, maxT: the frames the buffers are sized for, else 7 more than the longest utterance])
CASES = {
    "bidirectional_cluster_h512": (512, 2, 1, False, [40] * 6, 1),
    "bidirectional_tensor_core_h1024": (1024, 2, 1, False, [24] * 4, 2),
    "unidirectional_h256": (256, 3, 2, True, [30] * 5, 1),
    "dnn": (256, 2, -1, False, [30] * 5, None),
    "ragged_h128": (128, 3, 2, False, [37, 50, 21, 50, 8, 44, 3], 1),
    "one_frame_h512": (512, 2, 1, False, [1] * 4, 1),
    # half of maxT x maxB rows: the H x H contraction then needs more split-K room than at maxT x maxB (fewer row tiles
    # than SMs add partial sums), more than an area sized for the forward shapes at maxT x maxB alone would hold
    "half_rows_h512": (512, 2, 1, False, [100] * 32, 1, 200),
}


@pytest.mark.parametrize("name", list(CASES))
def test_forward_layout_probs_are_bit_identical_to_a_training_call(name, cuda):
    import nnets.brnnet as brnnet
    import nnets.rnnet as unirnnet
    from _ctcb import lib, check
    torch = cuda
    H, N, tl, uni, lens, kernel = CASES[name][:6]
    D, K, B = 41, 62, len(lens)
    maxT = CASES[name][6] if len(CASES[name]) > 6 else max(lens) + 7
    if len(CASES[name]) > 6:
        need = lib.ctcb_gemm_workspace_bytes
        at_max = max(need(maxT * B, n_out, n_in) for n_out, n_in in ((H, D), (H, H), (K, H)))
        assert need(max(lens) * B, H, H) > at_max
    if kernel is not None:
        plan = (ctypes.c_int32 * 8)()
        check(lib.ctcb_debug_sweep_plan(H, B, 1 if uni else 2, plan))
        assert plan[0] == kernel, list(plan)
    cls = (unirnnet if uni else brnnet).NNet
    datas, labelss = recipes.synth_batch(D, K, lens, [min(3, T) for T in lens], seed=H + B)
    np.random.seed(12)
    nt = cls(D, K, H, N, maxT, temporalLayer=tl, maxUtts=B, maxLabels=3)
    nt.initParams()
    nf = cls(D, K, H, N, maxT, temporalLayer=tl, maxUtts=B, train=False)
    nf.initParams()
    nf.params.copy_(nt.params)
    assert (nt.temporalLayer > 0) == (tl > 0)
    fwd_bytes = lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(nf._cfg), None)
    assert nf._ws.numel() == fwd_bytes < nt._ws.numel()

    Tmax = max(lens)
    nt._batch.pack(datas, labelss).upload()
    nt.costAndGradDevice(nt._batch, want_probs=True)                 # training call, training layout
    p_train = nt._probs_view(B, Tmax).clone()
    p_big = nt._forward_device(nt._batch).clone()                     # forward-only in the training-size workspace
    nf._batch.pack(datas, None).upload()
    p_fwd = nf.costAndGradDevice(nf._batch).clone()                   # forward-only in the forward-size workspace
    torch.cuda.synchronize()
    assert int(nf._errflag.item()) == 0 and int(nt._errflag.item()) == 0
    assert p_fwd.shape == (Tmax, B, K)
    assert np.isfinite(p_fwd.cpu().numpy()).all()
    a, b, c = (p.view(torch.int32).cpu().numpy() for p in (p_train, p_big, p_fwd))
    assert np.array_equal(a, c), "forward layout differs from the training call"
    assert np.array_equal(b, c), "forward layout in a training-size workspace differs"


def test_forward_batch_matches_oracle_in_input_order(cuda):
    """21 ragged utterances in shuffled order, micro-batches of 8, against the float64 oracle's forward pass
    (the 1e-5 absolute probability bound of test_brnn_gpu's forward-only check); a training net gives the same bits."""
    import nnets.brnnet as brnnet
    D, K, H, N, tl, maxT = 41, 62, 256, 2, 1, 60
    rng = np.random.RandomState(21)
    lens = [int(x) for x in rng.randint(1, maxT + 1, size=21)]
    lens[5] = maxT
    datas, _ = recipes.synth_batch(D, K, lens, [1] * 21, seed=21)
    np.random.seed(8)
    on = brnn_oracle.NNet(D, K, H, N, maxT, temporalLayer=tl, dtype=np.float64)
    on.initParams()
    np.random.seed(8)
    nn = brnnet.NNet(D, K, H, N, maxT, temporalLayer=tl, train=False, maxUtts=8)
    nn.initParams()
    got = nn.forwardBatch(datas)
    assert len(got) == 21
    worst = 0.0
    for d, p in zip(datas, got):
        assert p.dtype == np.float32 and p.shape == (K, d.shape[1]) and p.flags.c_contiguous
        worst = max(worst, float(np.abs(p - on.forward(d)[3]).max()))
    print(json.dumps({"forwardBatch_vs_oracle_max_abs_prob_err": worst}))
    assert worst < 1e-5, worst
    # one utterance at a time through the reference call gives the same probabilities per utterance (B differs, so
    # the plans may too: the oracle's bound, not bits)
    for d, p in list(zip(datas, got))[:3]:
        assert np.abs(nn.costAndGrad(d) - p).max() < 1e-5
    np.random.seed(8)
    nt = brnnet.NNet(D, K, H, N, maxT, temporalLayer=tl, maxUtts=8, maxLabels=4)
    nt.initParams()
    assert all(np.array_equal(a, b) for a, b in zip(nt.forwardBatch(datas), got))
    assert nn.forwardBatch([]) == []
    with pytest.raises(ValueError):
        nn.forwardBatch([datas[0], np.zeros((D, maxT + 1), dtype=np.float32)])


def _per_utterance_arks(loader, nn, fn, out_dir):
    """The writer as it was before forwardBatch: one costAndGrad(data) per key, then header and log-probabilities."""
    data_dict, _, keys, sizes = loader.loadDataFileDict(fn)
    lik = dict()
    with open(os.path.join(out_dir, "loglikelihoods%d.ark" % fn), "wb") as fid:
        for i, k in enumerate(keys):
            fid.write((k + ' ').encode() + struct.pack('b', 0) + b'BFM ' + struct.pack('b', 4)
                      + struct.pack('i', int(sizes[i])) + struct.pack('b', 4) + struct.pack('i', nn.outputDim))
            probs = nn.costAndGrad(data_dict[k])
            with np.errstate(divide='ignore'):
                probs = np.log(probs)
            probs.T.tofile(fid)
            lik[k] = probs
    with open(os.path.join(out_dir, "loglikelihoods_%d.pk" % fn), "wb") as f:
        pickle.dump(lik, f)


def _read_ark(path):
    """[(key, rows, cols, float32 rows x cols)] of a binary BFM ark."""
    buf, pos, out = open(path, "rb").read(), 0, []
    while pos < len(buf):
        sp = buf.index(b" ", pos)
        key = buf[pos:sp].decode()
        assert buf[sp + 1:sp + 6] == b"\x00BFM "
        rows, cols = struct.unpack("i", buf[sp + 7:sp + 11])[0], struct.unpack("i", buf[sp + 12:sp + 16])[0]
        pos = sp + 16 + 4 * rows * cols
        out.append((key, rows, cols, np.frombuffer(buf[sp + 16:pos], dtype=np.float32).reshape(rows, cols)))
    return out


# Largest |difference| of the log-likelihoods in [-80, 0] between maxUtts = 8 and the per-utterance loop: about 2.5e-6
# of the magnitude of the values near -80 (the plans of the contractions differ with B).  The bound is 4x that.  The
# line test_write_log_likes_batched_vs_per_utterance printed (pytest -s) on one H100 80GB HBM3, power limit 400 W:
#   {"loglik_maxUtts8_vs_loop_max_abs_diff": 0.0001983642578125, "neg_inf_entries": 14,
#    "finite_entries_below_-80": 132, "tolerance": 0.000792}
LOGLIK_MEASURED = 1.98e-4
LOGLIK_TOL = 4 * LOGLIK_MEASURED


def test_write_log_likes_batched_vs_per_utterance(cuda, tmp_path):
    import dataLoader as dl
    import nnets.brnnet as brnnet
    import writeLikelihoods
    data = str(tmp_path / "data") + "/"
    dl.write_synthetic_file(data, 1, num_utts=19, rawsize=20, outputDim=9, T_range=(5, 39), L_range=(3, 5))
    loader = dl.DataLoader(data, 20, 16, data)
    D, K, H, N, tl, maxT = 16, 9, 128, 3, 2, 40

    def net(maxUtts):
        np.random.seed(5)
        nn = brnnet.NNet(D, K, H, N, maxT, temporalLayer=tl, train=False, maxUtts=maxUtts)
        nn.initParams()
        nn.stack[N][0].mul_(30.0)       # logits spread over ~100: log-likelihoods below -80, and -inf
        return nn

    dirs = {n: tmp_path / n for n in ("loop", "one", "eight")}
    for d in dirs.values():
        d.mkdir()
    _per_utterance_arks(loader, net(1), 1, str(dirs["loop"]))
    writeLikelihoods.writeLogLikes(loader, net(1), 1, str(dirs["one"]), writePickle=True)
    writeLikelihoods.writeLogLikes(loader, net(8), 1, str(dirs["eight"]), writePickle=True)
    for f in ("loglikelihoods1.ark", "loglikelihoods_1.pk"):
        assert (dirs["one"] / f).read_bytes() == (dirs["loop"] / f).read_bytes(), f
    ref, got = _read_ark(str(dirs["loop"] / "loglikelihoods1.ark")), _read_ark(str(dirs["eight"] / "loglikelihoods1.ark"))
    assert [r[:3] for r in got] == [r[:3] for r in ref]
    pk_ref = pickle.load(open(str(dirs["loop"] / "loglikelihoods_1.pk"), "rb"))
    pk_got = pickle.load(open(str(dirs["eight"] / "loglikelihoods_1.pk"), "rb"))
    assert list(pk_got) == list(pk_ref)
    worst, n_inf, n_low = 0.0, 0, 0
    for (_, _, _, a), (_, _, _, b) in zip(got, ref):
        ia, ib = np.isneginf(a), np.isneginf(b)
        n_inf += int(ib.sum())
        assert not (ia & ~ib & ~(b < -80)).any() and not (ib & ~ia & ~(a < -80)).any()
        # below about -87 the softmax's exp leaves float32's normal range, and the last bits of a subnormal
        # probability are a large part of its logarithm: those entries are only required to be very small
        normal = ~ia & ~ib & (a >= -80) & (b >= -80)
        n_low += int((~ia & ~ib & ~normal).sum())
        worst = max(worst, float(np.abs(a[normal] - b[normal]).max()))
    print(json.dumps({"loglik_maxUtts8_vs_loop_max_abs_diff": worst, "neg_inf_entries": n_inf,
                      "finite_entries_below_-80": n_low, "tolerance": LOGLIK_TOL}))
    assert n_inf > 0 and n_low > 0         # the comparison sees both regimes
    assert worst <= LOGLIK_TOL, worst


def test_run_nnet_test_with_max_utts_writes_the_same_arks(cuda, tmp_path):
    import dataLoader as dl
    import runNNet
    data = str(tmp_path / "data") + "/"
    for fn in (1, 2):
        dl.write_synthetic_file(data, fn, num_utts=11, rawsize=20, outputDim=9, T_range=(10, 39), L_range=(3, 6))
    runNNet.run(["--layerSize", "64", "--numLayers", "2", "--temporalLayer", "1", "--epochs", "1", "--step", "1e-3",
                 "--dataDir", data, "--numFiles", "1", "--inputDim", "16", "--rawDim", "20", "--outputDim", "9",
                 "--maxUttLen", "40", "--maxLabels", "6", "--batchSize", "4", "--save_every", "1",
                 "--runDir", str(tmp_path / "runs"), "--quiet"])
    run_dir = os.path.join(str(tmp_path / "runs"), os.listdir(str(tmp_path / "runs"))[0])
    cfg = os.path.join(run_dir, "cfg.json")
    common = ["--cfg_file", cfg, "--test", "--dataDir", data, "--numFiles", "2"]
    nets = {}
    for name, extra in (("default", []), ("batched", ["--maxUtts", "8"])):
        nets[name] = runNNet.run(common + ["--outDir", str(tmp_path / name)] + extra)
    assert nets["default"].maxUtts == 1 and nets["batched"].maxUtts == 8
    for fn in (1, 2):
        a = _read_ark(str(tmp_path / "default" / ("loglikelihoods%d.ark" % fn)))
        b = _read_ark(str(tmp_path / "batched" / ("loglikelihoods%d.ark" % fn)))
        assert len(a) == 11 and [r[:3] for r in a] == [r[:3] for r in b]
