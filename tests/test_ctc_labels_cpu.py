"""The host boundaries of the CTC's label sequences, without a device: ctc_fast.ctc_loss raises IndexError for a label
outside [0, K) before it reaches the device, and NNet refuses such a label (ValueError naming the utterance and the label)
where it packs a minibatch.  The device-side check of the same contract is tests/test_ctc_labels_gpu.py."""
import numpy as np
import pytest

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


@pytest.mark.parametrize("bad", ["K", "K+1", "-1", "INT_MAX", "INT_MIN"])
@pytest.mark.parametrize("pos", [0, 2, 4])
def test_ctc_loss_refuses_labels_outside_the_classes(bad, pos):
    import ctc_fast
    K, T = 6, 9
    p = np.asfortranarray(np.full((K, T), 1.0 / K))
    seq = np.array([1, 2, 3, 4, 5], np.int32)
    seq[pos] = {"K": K, "K+1": K + 1, "-1": -1, "INT_MAX": INT_MAX, "INT_MIN": INT_MIN}[bad]
    with pytest.raises(IndexError):
        ctc_fast.ctc_loss(p, seq)


def test_ctc_loss_takes_the_edge_labels():
    """0 and K - 1 are labels: without a device the call gets as far as the device (RuntimeError), not IndexError."""
    import torch
    import ctc_fast
    if torch.cuda.is_available():
        pytest.skip("CUDA present: tests/test_ctc_labels_gpu.py runs these labels")
    K, T = 6, 9
    with pytest.raises(RuntimeError):
        ctc_fast.ctc_loss(np.asfortranarray(np.full((K, T), 1.0 / K)), np.array([0, K - 1, 0], np.int32))
    with pytest.raises(RuntimeError):
        ctc_fast.ctc_loss(np.asfortranarray(np.full((K, T), 1.0 / K)), np.zeros(0, np.int32))


@pytest.mark.parametrize("bad", [7, 8, -1, INT_MAX, INT_MIN])
def test_nnet_refuses_a_label_outside_the_classes(bad):
    import nnets.brnnet as brnnet
    K = 7
    seq = [3, 0, 6, bad, 2]
    with pytest.raises(ValueError) as e:
        brnnet.utterance_labels(4, seq, 10, K)
    msg = str(e.value)
    assert "utterance 4" in msg and "label %d" % bad in msg and "position 3" in msg, msg


def test_nnet_label_checks():
    import nnets.brnnet as brnnet
    l = brnnet.utterance_labels(0, [0, 6, 6, 1], 4, 7)
    assert l.dtype == np.int32 and l.tolist() == [0, 6, 6, 1]
    assert brnnet.utterance_labels(1, [], 4, 7).shape == (0,)
    with pytest.raises(ValueError, match="utterance 2 has 5 labels"):
        brnnet.utterance_labels(2, [1, 1, 1, 1, 1], 4, 7)
