"""CPU tests of batched inference: the forward-only workspace size (ctcb_brnn_forward_workspace_bytes), the rank -> file
rule of `runNNet --test` under torchrun (parallel.rank_files), and writeLogLikes over NNet.forwardBatch with a stub
net.  No compute call is made here."""
import ctypes
import io
import os
import pickle
import struct

import numpy as np
import pytest


def _cfg(D, K, H, N, tl, maxT, maxB, L, uni=0):
    import _ctcb
    return _ctcb.BrnnConfig(D, K, H, N, tl, maxT, maxB, L, 0.0, 20.0, uni)


def _sizes(cfg):
    import _ctcb
    off = ctypes.c_size_t(12345)
    fwd = _ctcb.lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(cfg), ctypes.byref(off))
    return fwd, off.value, _ctcb.lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg))


@pytest.mark.parametrize("kind", ["bidirectional", "unidirectional", "dnn"])
def test_forward_workspace_is_smaller_and_holds_the_error_flag(kind):
    import _ctcb
    tl, uni = {"bidirectional": (1, 0), "unidirectional": (1, 1), "dnn": (0, 0)}[kind]
    fwd, off, train = _sizes(_cfg(41, 62, 512, 2, tl, 200, 32, 30, uni))
    assert 0 < fwd < train
    assert off % 256 == 0 and off + 4 <= fwd
    # without the error-flag output the size is the same
    assert _ctcb.lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(_cfg(41, 62, 512, 2, tl, 200, 32, 30, uni)),
                                                       None) == fwd


def test_forward_workspace_sizes_of_the_layouts_differ_by_the_sweep_outputs():
    """Two slabs + For + Back (bi-directional) > two slabs + For (uni-directional) > two slabs (DNN)."""
    bi, uni, dnn = (_sizes(_cfg(41, 62, 512, 2, tl, 200, 32, 30, u))[0] for tl, u in ((1, 0), (1, 1), (0, 0)))
    assert bi > uni > dnn


def test_forward_workspace_invalid_config_is_zero():
    import _ctcb
    off = ctypes.c_size_t(7)
    bad = _cfg(0, 62, 512, 2, 1, 200, 32, 30)
    assert _ctcb.lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(bad), ctypes.byref(off)) == 0
    assert off.value == 7                       # left alone
    assert _ctcb.lib.ctcb_brnn_forward_workspace_bytes(None, None) == 0
    assert _ctcb.lib.ctcb_brnn_forward_workspace_bytes(ctypes.byref(_cfg(41, 62, 512, 2, 1, 200, 32, 600)), None) == 0


def test_forward_workspace_at_c4_widths_is_under_three_tenths_of_training():
    """C4 widths (H = 2048, N = 5, temporal layer 3, K = 35) at the reference's maxUttLen 5000 and 32 utterances: the
    layout arithmetic gives about 4H floats per frame-row against about 16H plus the CTC spill.  Without a device both
    sizes use the 132 SMs of the H100 SXM."""
    fwd, off, train = _sizes(_cfg(41, 35, 2048, 5, 3, 5000, 32, 150))
    ratio = fwd / float(train)
    print("C4 widths, maxT 5000, maxB 32: forward %.2f GB, training %.2f GB, ratio %.3f" % (fwd / 1e9, train / 1e9, ratio))
    assert ratio <= 0.3, ratio


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_rank_files_cover_every_file_once(world):
    import parallel
    for start, num in ((1, 1), (1, 7), (3, 10), (5, 4)):
        got = [parallel.rank_files(start, num, r, world) for r in range(world)]
        flat = sorted(f for fs in got for f in fs)
        assert flat == list(range(start, num + 1)), (start, num, world, got)
        for r, fs in enumerate(got):
            assert fs == list(range(start + r, num + 1, world))


class _StubNet(object):
    """What writeLogLikes needs of a net: forwardBatch, maxBatch, outputDim.  Probabilities are a softmax of a
    fixed projection of the features with exact zeros in some places (log -> -inf)."""

    def __init__(self, D, K, maxBatch):
        rng = np.random.RandomState(3)
        self.W = rng.randn(K, D)
        self.outputDim, self.maxBatch = K, maxBatch
        self.calls = []

    def probs(self, d):
        z = self.W.dot(d)
        e = np.exp(z - z.max(axis=0))
        p = (e / e.sum(axis=0)).astype(np.float32)
        p[0, ::3] = 0.0
        return p

    def forwardBatch(self, datas):
        self.calls.append(len(datas))
        return [self.probs(d) for d in datas]


class _StubLoader(object):
    def __init__(self, D, lens):
        rng = np.random.RandomState(4)
        self.keys = ["utt%d_%04d" % (7, i) for i in range(len(lens))]
        self.data = {k: rng.randn(D, T).astype(np.float32) for k, T in zip(self.keys, lens)}

    def loadDataFileDict(self, fn):
        return self.data, {k: [1, 2] for k in self.keys}, list(self.keys), [self.data[k].shape[1] for k in self.keys]


def _per_key_loop(loader, nn, fn):
    """The reference's loop (analysis-utils/writeLikelihoods.py): header, then log(probs).T of each key in turn."""
    data_dict, _, keys, sizes = loader.loadDataFileDict(fn)
    ark, lik = io.BytesIO(), dict()
    for i, k in enumerate(keys):
        ark.write((k + ' ').encode() + struct.pack('b', 0) + b'BFM ' + struct.pack('b', 4) + struct.pack('i', int(sizes[i]))
                  + struct.pack('b', 4) + struct.pack('i', nn.outputDim))
        with np.errstate(divide='ignore'):
            p = np.log(nn.probs(data_dict[k]))
        ark.write(p.T.tobytes())
        lik[k] = p
    return ark.getvalue(), pickle.dumps(lik)


def test_write_log_likes_matches_the_per_key_loop(tmp_path):
    import writeLikelihoods
    D, K = 6, 5
    loader = _StubLoader(D, [7, 3, 12, 1, 9, 7])
    nn = _StubNet(D, K, 20)
    lik = writeLikelihoods.writeLogLikes(loader, nn, 7, str(tmp_path), writePickle=True)
    assert nn.calls == [6]                      # the whole file in one call, the net cuts its own micro-batches
    ark, pk = _per_key_loop(loader, nn, 7)
    assert open(os.path.join(str(tmp_path), "loglikelihoods7.ark"), "rb").read() == ark
    assert open(os.path.join(str(tmp_path), "loglikelihoods_7.pk"), "rb").read() == pk
    assert list(lik) == loader.keys and np.isneginf(lik[loader.keys[0]]).any()


def test_write_log_likes_keeps_the_length_assertion(tmp_path):
    import writeLikelihoods
    loader = _StubLoader(4, [5, 20])
    nn = _StubNet(4, 3, 20)
    with pytest.raises(AssertionError, match="Need larger max utt length"):
        writeLikelihoods.writeLogLikes(loader, nn, 1, str(tmp_path))
    assert nn.calls == []
