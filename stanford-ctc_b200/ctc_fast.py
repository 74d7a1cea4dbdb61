"""ctc_fast -- drop-in for the reference's Cython module of the same name
(ctc_fast/ctc-loss/ctc_fast.pyx), computed on the H100 by libctcb200.

    ctc_loss(params, seq, blank=0)        -> (nll, grad, skip)      ctc_fast.pyx:13-152
    decode_best_path(probs, blank=0)      -> (hyp, align)           ctc_fast.pyx:154-187

Both keep the reference's argument contract (params: K x T float64 Fortran-contiguous ndarray of
per-frame probability distributions, seq: int32 labels) and error behaviour (ValueError for a
non-Fortran array; numerical infeasibility is reported through skip=True, never raised).
Where the reference's own float64 arithmetic runs out of range (long utterances with unaligned outputs) the
results differ from it on purpose: occupancies the reference loses to underflow (its gradient rows left at p)
are computed, and an utterance whose scaled trellis lost mass (where the reference returns a wrong loss) is
reported as skip=True with a zero gradient.  DESIGN.md section 4 has the measurements.
The batched, zero-copy entry `ctc_loss_batch` is what nnets.brnnet uses internally through the
C ABI; it is exported for callers that already hold activations on the device.
"""
import numpy as np

import _ctcb
from _ctcb import lib, check, ptr


def _check_params(params):
    if params is None:
        raise TypeError("Argument 'params' must not be None")
    if not isinstance(params, np.ndarray) or params.ndim != 2:
        raise ValueError("Buffer has wrong number of dimensions (expected 2)")
    if params.dtype != np.float64:
        raise ValueError("Buffer dtype mismatch, expected 'double' but got '%s'" % params.dtype)
    if not params.flags.f_contiguous:
        raise ValueError("ndarray is not Fortran contiguous")


def ctc_loss_batch(acts, T_per_utt, labels, label_off, max_labels, blank=0, is_prob=False,
                   utt_stride=None, frame_stride=None, grad=None, workspace=None):
    """Batched CTC on device tensors.  acts: float32 CUDA tensor holding B utterances of up to Tmax
    frames x K classes; default layout [B][Tmax][K] (pass strides, in elements, for time-major data).
    T_per_utt/labels/label_off: int32 CUDA tensors.  Returns (nll[B], grad like acts, skip[B]) on the
    device without synchronising."""
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
    nbytes = lib.ctcb_ctc_workspace_bytes(B, Tmax, int(max_labels))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=acts.device)
    nll = torch.empty(B, dtype=torch.float32, device=acts.device)
    skip = torch.empty(B, dtype=torch.int32, device=acts.device)
    check(lib.ctcb_ctc_loss_grad_f32(ptr(acts), int(bool(is_prob)), int(utt_stride), int(frame_stride), ptr(labels),
                                     ptr(label_off), ptr(T_per_utt), B, Tmax, K, int(max_labels), int(blank),
                                     ptr(grad), ptr(nll), ptr(skip), ptr(workspace), workspace.numel(),
                                     _ctcb.current_stream()))
    return nll, grad, skip


_scratch = {}


def _single_utterance_buffers(torch, dev, T, K, L):
    """Device and pinned-host buffers of the reference-signature call, kept per (T, K, |l|): a reference user who steps
    one utterance at a time (sgd.py:70-161) re-uses them instead of allocating seven tensors per call."""
    key = (dev.index, T, K, L)
    b = _scratch.get(key)
    if b is None:
        if len(_scratch) > 64:
            _scratch.clear()
        n_int = 3 + max(L, 1)                               # label_off[2], T, labels
        b = dict(h_acts=torch.empty(T * K, dtype=torch.float32).pin_memory(),
                 h_int=torch.empty(n_int, dtype=torch.int32).pin_memory(),
                 h_grad=torch.empty(T * K, dtype=torch.float32).pin_memory(),
                 h_out=torch.empty(2, dtype=torch.float32).pin_memory(),
                 d_acts=torch.empty(T * K, dtype=torch.float32, device=dev),
                 d_int=torch.empty(n_int, dtype=torch.int32, device=dev),
                 d_grad=torch.empty(T * K, dtype=torch.float32, device=dev),
                 d_out=torch.empty(2, dtype=torch.float32, device=dev),      # nll, skip (int32 bits)
                 ws=torch.empty(max(lib.ctcb_ctc_workspace_bytes(1, T, L), 1), dtype=torch.uint8, device=dev))
        _scratch[key] = b
    return b


def ctc_loss(params, seq, blank=0):
    """CTC loss function (reference signature).  params - n x m matrix of n-D probability
    distributions over m frames, Fortran order; seq - label ids.  Returns (objective, gradient with
    respect to the unnormalised inputs, skip).  Two H2D copies, one kernel, two D2H copies, ONE synchronisation."""
    _check_params(params)
    if seq is None:
        raise TypeError("Argument 'seq' must not be None")
    seq = np.ascontiguousarray(seq)
    if seq.dtype != np.int32 or seq.ndim != 1:
        raise ValueError("Buffer dtype mismatch, expected 'int' but got '%s'" % seq.dtype)
    torch = _ctcb.require_cuda()
    K, T = params.shape
    L = int(seq.shape[0])
    dev = torch.device("cuda", torch.cuda.current_device())
    b = _single_utterance_buffers(torch, dev, T, K, L)
    # K x T Fortran == T x K row-major: the frame-contiguous layout the kernel streams
    b["h_acts"].numpy().reshape(T, K)[...] = params.T
    hi = b["h_int"].numpy()
    hi[0], hi[1], hi[2] = 0, L, T
    hi[3:3 + L] = seq
    b["d_acts"].copy_(b["h_acts"], non_blocking=True)
    b["d_int"].copy_(b["h_int"], non_blocking=True)
    d_int, d_out = b["d_int"], b["d_out"]
    check(lib.ctcb_ctc_loss_grad_f32(ptr(b["d_acts"]), 1, T * K, K, d_int.data_ptr() + 12, d_int.data_ptr(),
                                     d_int.data_ptr() + 8, 1, T, K, L, int(blank), ptr(b["d_grad"]), d_out.data_ptr(),
                                     d_out.data_ptr() + 4, ptr(b["ws"]), b["ws"].numel(), _ctcb.current_stream()))
    b["h_grad"].copy_(b["d_grad"], non_blocking=True)
    b["h_out"].copy_(d_out, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    out = b["h_out"].numpy()
    g = b["h_grad"].numpy().reshape(T, K).astype(np.float64)
    return float(out[0]), np.asfortranarray(g.T), bool(out[1:2].view(np.int32)[0] != 0)


def decode_best_path(probs, blank=0):
    """Best path: most likely label per frame, collapse repeats, drop blanks and (as the reference
    does, ctc_fast.pyx:176-179) the SWBD noise labels 1, 2 and 8.  Returns (hyp, align)."""
    _check_params(probs)
    torch = _ctcb.require_cuda()
    K, T = probs.shape
    dev = torch.device("cuda", torch.cuda.current_device())
    acts = torch.from_numpy(np.ascontiguousarray(probs.T, dtype=np.float32)).to(dev)
    tl = torch.tensor([T], dtype=torch.int32, device=dev)
    hyp = torch.empty(T, dtype=torch.int32, device=dev)
    ali = torch.empty(T, dtype=torch.int32, device=dev)
    n = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.ctcb_ctc_best_path_f32(ptr(acts), T * K, K, ptr(tl), 1, T, K, int(blank), 1, ptr(hyp), ptr(ali),
                                     ptr(n), _ctcb.current_stream()))
    n = int(n.item())
    return hyp[:n].cpu().tolist(), ali[:n].cpu().tolist()
