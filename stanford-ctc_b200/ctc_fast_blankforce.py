"""ctc_fast_blankforce -- drop-in for the reference's second Cython CTC module
(ctc_fast/ctc-loss/ctc_fast_blankforce.pyx), computed on the H100 by libctcb200.

    ctc_loss(params, seq)                 -> (nll, grad, skip)      ctc_fast_blankforce.pyx:13-113
    decode_best_path(probs, blank=0)      -> hyp                    ctc_fast_blankforce.pyx:115-142

`seq` already contains the blanks (one trellis state per entry, at most 1024); see
csrc/ctc_blankforce.cu for the recursion.  Argument contract and error behaviour follow ctc_fast.py.
"""
import numpy as np

import _ctcb
from _ctcb import lib, check, ptr
from ctc_fast import _check_params


def ctc_loss_batch(acts, T_per_utt, seq, seq_off, max_states, is_prob=False, utt_stride=None, frame_stride=None,
                   grad=None, workspace=None):
    """Batched form on device tensors (layout and return values as ctc_fast.ctc_loss_batch).  Utterance u's states are
    seq[seq_off[u]:seq_off[u+1]].  The device checks each utterance before it reads its states: no frame, no state, more
    than max_states states, or a label outside [0, K) gives skip = 1 with a zero gradient."""
    torch = _ctcb.require_cuda()
    assert acts.is_cuda and acts.dtype == torch.float32 and acts.is_contiguous()
    B = T_per_utt.numel()
    K = acts.shape[-1]
    if utt_stride is None:
        Tmax = acts.shape[1]
        utt_stride, frame_stride = Tmax * K, K
    else:
        Tmax = acts.numel() // (B * K)
    if grad is None:
        grad = torch.empty_like(acts)
    nbytes = lib.ctcb_ctc_blankforce_workspace_bytes(B, Tmax, int(max_states))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=acts.device)
    nll = torch.empty(B, dtype=torch.float32, device=acts.device)
    skip = torch.empty(B, dtype=torch.int32, device=acts.device)
    check(lib.ctcb_ctc_blankforce_loss_grad_f32(ptr(acts), int(bool(is_prob)), int(utt_stride), int(frame_stride),
                                                ptr(seq), ptr(seq_off), ptr(T_per_utt), B, Tmax, K, int(max_states),
                                                ptr(grad), ptr(nll), ptr(skip), ptr(workspace), workspace.numel(),
                                                _ctcb.current_stream()))
    return nll, grad, skip


def ctc_loss(params, seq):
    """CTC loss function (reference signature): params K x T float64 Fortran order, seq int32 WITH blanks."""
    _check_params(params)
    if seq is None:
        raise TypeError("Argument 'seq' must not be None")
    seq = np.ascontiguousarray(seq)
    if seq.dtype != np.int32 or seq.ndim != 1:
        raise ValueError("Buffer dtype mismatch, expected 'int' but got '%s'" % seq.dtype)
    K, T = params.shape
    if seq.size == 0 or seq.min() < 0 or seq.max() >= K:
        raise IndexError("label sequence empty or out of range")     # the reference would read out of bounds
    torch = _ctcb.require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    acts = torch.from_numpy(np.ascontiguousarray(params.T, dtype=np.float32)).to(dev).view(1, T, K)
    lab = torch.from_numpy(seq).to(dev)
    off = torch.tensor([0, seq.shape[0]], dtype=torch.int32, device=dev)
    tl = torch.tensor([T], dtype=torch.int32, device=dev)
    nll, grad, skip = ctc_loss_batch(acts, tl, lab, off, seq.shape[0], is_prob=True)
    g = grad.view(T, K).cpu().numpy().astype(np.float64)
    return float(nll.item()), np.asfortranarray(g.T), bool(skip.item())


def decode_best_path(probs, blank=0):
    """Most likely label per frame, repeats and blanks removed; returns the hypothesis only."""
    _check_params(probs)
    torch = _ctcb.require_cuda()
    K, T = probs.shape
    dev = torch.device("cuda", torch.cuda.current_device())
    acts = torch.from_numpy(np.ascontiguousarray(probs.T, dtype=np.float32)).to(dev)
    tl = torch.tensor([T], dtype=torch.int32, device=dev)
    hyp = torch.empty(T, dtype=torch.int32, device=dev)
    ali = torch.empty(T, dtype=torch.int32, device=dev)
    n = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.ctcb_ctc_best_path_f32(ptr(acts), T * K, K, ptr(tl), 1, T, K, int(blank), 0, ptr(hyp), ptr(ali),
                                     ptr(n), _ctcb.current_stream()))
    return hyp[:int(n.item())].cpu().tolist()
