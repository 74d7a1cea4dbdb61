"""oracle/ctc_oracle.py -- TEST INFRASTRUCTURE ONLY.

ctypes front-end of oracle/ctc_oracle.c (the float64 C restatement of
ctc_fast/ctc-loss/ctc_fast.pyx:13-187 and ctc_fast_blankforce.pyx:13-142) plus a loader for oracle/_ref (the
reference's own .pyx compiled unmodified by oracle/build_ref.py).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (stanford-ctc_b200/) never does.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib_path():
    return os.path.join(HERE, "_build", "libctc_oracle.so")


def build(force=False):
    """gcc the C restatement into oracle/_build/ (git-ignored)."""
    src = os.path.join(HERE, "ctc_oracle.c")
    out = lib_path()
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if force or not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", src, "-o", out, "-lm"])
    return out


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.ctc_oracle_loss.restype = ctypes.c_int
        _LIB.ctc_oracle_loss.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        _LIB.ctc_oracle_loss_fb.restype = ctypes.c_int
        _LIB.ctc_oracle_loss_fb.argtypes = _LIB.ctc_oracle_loss.argtypes + [ctypes.c_void_p]
        _LIB.ctc_oracle_loss_log.restype = ctypes.c_int
        _LIB.ctc_oracle_loss_log.argtypes = _LIB.ctc_oracle_loss.argtypes
        _LIB.ctc_oracle_best_path.restype = ctypes.c_int
        _LIB.ctc_oracle_best_path.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_void_p]
        _LIB.ctc_oracle_loss_blankforce.restype = ctypes.c_int
        _LIB.ctc_oracle_loss_blankforce.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        _LIB.ctc_oracle_loss_blankforce_log.restype = ctypes.c_int
        _LIB.ctc_oracle_loss_blankforce_log.argtypes = _LIB.ctc_oracle_loss_blankforce.argtypes
        _LIB.ctc_oracle_best_path_blankforce.restype = ctypes.c_int
        _LIB.ctc_oracle_best_path_blankforce.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                         ctypes.c_void_p]
    return _LIB


def _call(fn, params, seq, blank, *extra):
    if not (isinstance(params, np.ndarray) and params.dtype == np.float64 and params.ndim == 2
            and params.flags.f_contiguous):
        raise ValueError("ndarray is not Fortran contiguous")
    seq = np.ascontiguousarray(seq, dtype=np.int32)
    K, T = params.shape
    grad = np.zeros((K, T), dtype=np.float64, order="F")
    nll = ctypes.c_double(0.0)
    skip = fn(params.ctypes.data, K, T, seq.ctypes.data, seq.shape[0], int(blank), grad.ctypes.data,
              ctypes.addressof(nll), *extra)
    return nll.value, grad, bool(skip)


def ctc_loss(params, seq, blank=0):
    """Same contract as the reference ctc_loss (ctc_fast.pyx:13-14,152): params K x T float64
    Fortran-contiguous, seq int32; returns (nll, grad K x T float64 F-order, skip)."""
    return _call(_lib().ctc_oracle_loss, params, seq, blank)


def ctc_loss_fb(params, seq, blank=0):
    """ctc_loss, plus the llBackward the reference computes and discards: (nll, grad, skip, llBackward).
    -nll == llBackward up to rounding unless the per-frame normalised trellis lost mass to underflow."""
    llb = ctypes.c_double(0.0)
    nll, grad, skip = _call(_lib().ctc_oracle_loss_fb, params, seq, blank, ctypes.addressof(llb))
    return nll, grad, skip, llb.value


def ctc_loss_log(params, seq, blank=0):
    """The same contract computed in the log domain (float64 log-sum-exp, no per-frame scaling): correct where the
    reference's products of normalised alpha and beta leave float64's range (long, unaligned utterances)."""
    return _call(_lib().ctc_oracle_loss_log, params, seq, blank)


def decode_best_path(probs, blank=0):
    probs = np.asfortranarray(probs, dtype=np.float64)
    K, T = probs.shape
    hyp = np.zeros(T, dtype=np.int32)
    align = np.zeros(T, dtype=np.int32)
    n = _lib().ctc_oracle_best_path(probs.ctypes.data, K, T, int(blank), hyp.ctypes.data, align.ctypes.data)
    return hyp[:n].tolist(), align[:n].tolist()


def _call_bf(fn, params, seq):
    if not (isinstance(params, np.ndarray) and params.dtype == np.float64 and params.ndim == 2
            and params.flags.f_contiguous):
        raise ValueError("ndarray is not Fortran contiguous")
    seq = np.ascontiguousarray(seq, dtype=np.int32)
    K, T = params.shape
    grad = np.zeros((K, T), dtype=np.float64, order="F")
    nll = ctypes.c_double(0.0)
    skip = fn(params.ctypes.data, K, T, seq.ctypes.data, seq.shape[0], grad.ctypes.data, ctypes.addressof(nll))
    return nll.value, grad, bool(skip)


def ctc_loss_blankforce(params, seq):
    """ctc_fast_blankforce.pyx:13-113 restated (oracle/ctc_oracle.c): seq already holds the blanks."""
    return _call_bf(_lib().ctc_oracle_loss_blankforce, params, seq)


def ctc_loss_blankforce_log(params, seq):
    """The blank-forced contract in the log domain (float64 log-sum-exp, no per-frame scaling): correct where the
    reference's normalised trellises underflow (long, unaligned utterances).  An empty seq or T = 0 is skip."""
    return _call_bf(_lib().ctc_oracle_loss_blankforce_log, params, seq)


def decode_best_path_blankforce(probs, blank=0):
    """ctc_fast_blankforce.pyx:115-142: returns the hypothesis only."""
    probs = np.asfortranarray(probs, dtype=np.float64)
    K, T = probs.shape
    hyp = np.zeros(T, dtype=np.int32)
    n = _lib().ctc_oracle_best_path_blankforce(probs.ctypes.data, K, T, int(blank), hyp.ctypes.data)
    return hyp[:n].tolist()


# ---------------------------------------------------------------------------------------------
# oracle/_ref: the unmodified reference extension (kind "reference")
# ---------------------------------------------------------------------------------------------
_REF = {}


def ref_module(name="ctc_fast"):
    """Import a compiled reference module (ctc_fast | ctc_fast_blankforce) from oracle/_ref; None if
    it was never built."""
    if name not in _REF:
        import importlib.util
        import sysconfig
        so = os.path.join(HERE, "_ref", name + sysconfig.get_config_var("EXT_SUFFIX"))
        if not os.path.exists(so):
            return None
        # The extension's init symbol is PyInit_<name>, so it must be loaded under that name; keep it
        # OUT of sys.modules so that `import ctc_fast` still resolves to the product's drop-in module.
        prev = sys.modules.get(name)
        spec = importlib.util.spec_from_file_location(name, so)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        if prev is not None:
            sys.modules[name] = prev
        else:
            sys.modules.pop(name, None)
        _REF[name] = mod
    return _REF[name]


def ref_ctc_loss_blankforce(params, seq):
    """The unmodified ctc_fast_blankforce.ctc_loss; failure path mapped as in ref_ctc_loss."""
    mod = ref_module("ctc_fast_blankforce")
    if mod is None:
        raise RuntimeError("oracle/_ref not built (run oracle/build_ref.py with CTC_REFERENCE_DIR set)")
    try:
        nll, grad, skip = mod.ctc_loss(params, np.ascontiguousarray(seq, dtype=np.int32))
        return float(nll), grad, bool(skip)
    except (AttributeError, ZeroDivisionError, FloatingPointError):
        return float("nan"), np.zeros(params.shape, dtype=np.float64, order="F"), True


def ref_ctc_loss(params, seq, blank=0):
    """Call the unmodified reference.  Its failure path does `print e.message`
    (ctc_fast.pyx:148), which under Python 3 raises AttributeError out of the handler instead of
    returning skip=True -- map that (and a bare ZeroDivisionError) to skip=True with zero grad."""
    mod = ref_module()
    if mod is None:
        raise RuntimeError("oracle/_ref not built (run oracle/build_ref.py with CTC_REFERENCE_DIR set)")
    try:
        nll, grad, skip = mod.ctc_loss(params, np.ascontiguousarray(seq, dtype=np.int32), blank)
        return float(nll), grad, bool(skip)
    except (AttributeError, ZeroDivisionError, FloatingPointError):
        return float("nan"), np.zeros(params.shape, dtype=np.float64, order="F"), True
