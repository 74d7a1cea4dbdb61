"""CPU tests of the drop-in boundary: libctcb200.so loads, exports every symbol include/ctcb200.h
declares, and its host-side (no-GPU) entry points behave.  No compute call is made here."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "ctcb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ctcb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import _ctcb
    names = _declared()
    assert len(names) >= 18
    for n in names:
        assert hasattr(_ctcb.lib, n), "libctcb200.so does not export %s" % n
    assert set(names) == set(_ctcb.EXPORTS), "binding table and header disagree"
    assert _ctcb.lib.ctcb_version() >= 100


def test_header_cites_reference_interfaces():
    src = open(os.path.join(ROOT, "include", "ctcb200.h")).read()
    for cite in ("ctc_fast.pyx:13-152", "ctc_fast.pyx:154-187", "brnnet.py:10-277", "sgd.py:91-161",
                 "ctc_fast_blankforce.pyx:13-113", "rnnet.py:91-191", "nnet.py:57-113"):
        assert cite in src


def test_param_layout_matches_reference_stack():
    """Flat layout = the reference's stack order with its shapes (brnnet.py:38-41,66-72)."""
    import _ctcb
    cfg = _ctcb.BrnnConfig(41, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0)
    nt = _ctcb.lib.ctcb_brnn_num_tensors(ctypes.byref(cfg))
    assert nt == 2 * 3 + 4
    shapes, offs = [], []
    off, r, c = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    for i in range(nt):
        assert _ctcb.lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), i, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
        shapes.append((r.value, c.value)); offs.append(off.value)
    assert shapes == [(512, 41), (512, 1), (512, 512), (512, 1), (62, 512), (62, 1),
                      (512, 512), (1, 1), (512, 512), (1, 1)]
    assert all(o % 4 == 0 for o in offs) and offs == sorted(offs)
    n = _ctcb.lib.ctcb_brnn_param_count(ctypes.byref(cfg))
    assert n >= sum(a * b for a, b in shapes) and n % 4 == 0
    assert _ctcb.lib.ctcb_brnn_workspace_bytes(ctypes.byref(cfg)) > 0
    # temporalLayer >= numLayers+1 or <= 0 -> no temporal tensors
    cfg2 = _ctcb.BrnnConfig(41, 62, 512, 2, 0, 200, 32, 30, 0.0, 20.0)
    assert _ctcb.lib.ctcb_brnn_num_tensors(ctypes.byref(cfg2)) == 6
    # uni-directional: one recurrent matrix + its dummy bias (rnnet.py:57-65)
    cfg3 = _ctcb.BrnnConfig(41, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0, 1)
    assert _ctcb.lib.ctcb_brnn_num_tensors(ctypes.byref(cfg3)) == 8
    assert _ctcb.lib.ctcb_brnn_tensor_info(ctypes.byref(cfg3), 6, ctypes.byref(off), ctypes.byref(r), ctypes.byref(c)) == 0
    assert (r.value, c.value) == (512, 512)
    assert _ctcb.lib.ctcb_ctc_blankforce_workspace_bytes(4, 100, 61) == 4 * 100 * 61 * 8
    assert _ctcb.lib.ctcb_ctc_blankforce_workspace_bytes(4, 100, 1025) == 0


def test_error_reporting():
    import _ctcb
    cfg = _ctcb.BrnnConfig(41, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0)
    rc = _ctcb.lib.ctcb_brnn_tensor_info(ctypes.byref(cfg), 99, None, None, None)
    assert rc == -1 and b"out of range" in _ctcb.lib.ctcb_last_error()
    with pytest.raises(ValueError):
        _ctcb.check(rc)
    bad = _ctcb.BrnnConfig(0, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0)
    h = ctypes.c_void_p()
    assert _ctcb.lib.ctcb_brnn_create(ctypes.byref(bad), ctypes.byref(h)) == -1
    assert _ctcb.lib.ctcb_ctc_workspace_bytes(4, 100, 600) == 0          # > 511 labels: unsupported
    # the CTC kernel selector takes 0..4 (automatic, warp, pair, par, ckpt) and nothing else
    assert _ctcb.lib.ctcb_debug_set_ctc_kernel(7) == -1 and b"not in 0..4" in _ctcb.lib.ctcb_last_error()
    assert _ctcb.lib.ctcb_debug_set_ctc_kernel(0) == 0
    # fp64 trellis rows [T][64] + one (even-padded) word per 16-frame tile; two planes for small batches (alpha and beta)
    assert _ctcb.lib.ctcb_ctc_workspace_bytes(4, 100, 30) == 4 * (100 * 64 + 8) * 8 * 2
    assert _ctcb.lib.ctcb_ctc_workspace_bytes(1000, 100, 30) == 1000 * (100 * 64 + 8) * 8


def test_gemm_row_limit():
    """Both contraction kernels put 128-row output tiles on gridDim.y: M beyond 65,535 tiles is refused before anything
    is read or launched, and so is a net whose maxT * maxB rows would need such a contraction."""
    import _ctcb
    lib = _ctcb.lib
    limit = 128 * 65535
    buf = (ctypes.c_float * 4)()
    p = ctypes.addressof(buf)
    assert lib.ctcb_gemm_f32(0, 1, limit + 1, 1, 1, 1.0, p, 1, p, 1, 0.0, p, 1, None, 0, None, None, 0, None) == -1
    assert b"exceeds" in lib.ctcb_last_error()
    assert lib.ctcb_gemm_pair_f32(1, 0, limit + 1, 1, 1, 1.0, p, p, limit + 1, p, p, 1, 0.0, p, p, 1, None, 0,
                                  None) == -1
    assert b"exceeds" in lib.ctcb_last_error()
    ok = _ctcb.BrnnConfig(41, 62, 16, 2, 1, 1000, limit // 1000, 30, 0.0, 20.0)
    over = _ctcb.BrnnConfig(41, 62, 16, 2, 1, 1000, limit // 1000 + 1, 30, 0.0, 20.0)
    assert lib.ctcb_brnn_param_count(ctypes.byref(ok)) > 0
    assert lib.ctcb_brnn_param_count(ctypes.byref(over)) <= 0
    h = ctypes.c_void_p()
    assert lib.ctcb_brnn_create(ctypes.byref(over), ctypes.byref(h)) == -1
    assert b"rows exceed" in lib.ctcb_last_error()


def test_step_reduction_entry_points_check_their_arguments():
    """ctcb_colsum_f32, ctcb_debug_colsum_plan and ctcb_softmax_rows_f32 refuse bad arguments before any launch, and the
    delta hook (what = 7) refuses the maps it cannot expose."""
    import _ctcb
    lib = _ctcb.lib
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    aligned = (p + 15) // 16 * 16
    assert lib.ctcb_colsum_workspace_bytes(1000, 5) == 8 * 5 * 4
    assert lib.ctcb_colsum_workspace_bytes(0, 5) == 0 and lib.ctcb_colsum_workspace_bytes(5, 0) == 0
    need = lib.ctcb_colsum_workspace_bytes(3, 4)
    for args in ((None, 3, 4, p, 0, aligned, need), (p, 3, 4, None, 0, aligned, need), (p, 3, 4, p, 0, None, need),
                 (p, 0, 4, p, 0, aligned, need), (p, -1, 4, p, 0, aligned, need), (p, 3, 0, p, 0, aligned, need),
                 (p, 3, -4, p, 0, aligned, need), (p, 128 * 65535 + 1, 4, p, 0, aligned, 1 << 40),
                 (p, 3, 4, p, 0, aligned + 4, need)):
        assert lib.ctcb_colsum_f32(*args, None) == -1, args
    assert lib.ctcb_colsum_f32(p, 3, 4, p, 1, aligned, need - 1, None) == -3
    assert b"workspace" in lib.ctcb_last_error()
    out = (ctypes.c_int32 * 4)()
    assert lib.ctcb_debug_colsum_plan(0, 4, aligned, out) == -1
    assert lib.ctcb_debug_colsum_plan(3, 0, aligned, out) == -1
    assert lib.ctcb_debug_colsum_plan(3, 4, aligned, None) == -1
    assert lib.ctcb_debug_colsum_plan(5, 64, aligned, out) == 0 and list(out)[0] == 1 and list(out)[2] == 128
    assert lib.ctcb_debug_colsum_plan(5, 64, aligned + 4, out) == 0 and list(out) == [0, 2, 1024, 1]
    assert lib.ctcb_debug_colsum_plan(5000, 35, aligned, out) == 0 and list(out) == [0, 2, 1024, 5]
    for args in ((None, p, 3, 4), (p, None, 3, 4), (p, p, 0, 4), (p, p, -3, 4), (p, p, 3, 0), (p, p, 3, -1)):
        assert lib.ctcb_softmax_rows_f32(*args, None) == -1, args
    # the delta of map `layer`: 1..N+1 only, G wide at an LSTM layer, refused above the lowest two layers of a
    # uni-directional clipped-ReLU stack (the pair they share is overwritten)
    off, width = ctypes.c_size_t(), ctypes.c_int32()
    hook = lambda cfg, layer: lib.ctcb_brnn_activation_offset(ctypes.byref(cfg), 7, layer, ctypes.byref(off),  # noqa: E731
                                                              ctypes.byref(width))
    bi = _ctcb.BrnnConfig(41, 62, 512, 2, 1, 200, 32, 30, 0.0, 20.0)
    assert hook(bi, 0) == -1 and hook(bi, 4) == -1
    assert [hook(bi, j) == 0 and width.value for j in (1, 2, 3)] == [512, 512, 62]
    lstm = _ctcb.BrnnConfig(41, 62, 64, 2, 1, 200, 32, 30, 0.0, 20.0, 0, 1, 1)
    assert hook(lstm, 1) == 0 and width.value == 2 * 4 * 64
    uni3 = _ctcb.BrnnConfig(41, 62, 64, 4, 1, 200, 32, 30, 0.0, 20.0, 1, 3)
    seen = set()
    for j in (1, 2, 4, 5):
        assert hook(uni3, j) == 0 and width.value == (62 if j == 5 else 64), j
        seen.add(off.value)
    assert len(seen) == 4
    assert hook(uni3, 3) == -1 and b"overwritten" in lib.ctcb_last_error()
    uni3_lstm = _ctcb.BrnnConfig(41, 62, 64, 4, 1, 200, 32, 30, 0.0, 20.0, 1, 3, 1)
    assert hook(uni3_lstm, 3) == 0 and width.value == 4 * 64


# The knobs of INTEGRATION.md section 4 that ctcb_debug_set_knob takes: every documented value, and a value outside them
KNOBS = {"CTCB_GEMM": (["simt"], "s"), "CTCB_GEMM_TC_COPY": (["0", "1"], "2"), "CTCB_GEMM_TRACE": (["1"], "0"),
         "CTCB_SWEEP": (["auto", "barrier", "reread"], "b"), "CTCB_SWEEP_NB": ([str(n) for n in range(1, 9)], "9"),
         "CTCB_SWEEP_TC": (["0", "1", "2"], "3"), "CTCB_SWEEP_TC_CS": (["1", "2", "4"], "3"),
         "CTCB_SWEEP_TC_COOP": (["0"], "1"), "CTCB_SWEEP_TRACE": (["1"], "0"),
         "CTCB_CTC": (["auto", "warp", "pair", "par", "ckpt"], "pa"), "CTCB_LSTM": (["auto", "reread"], "reg"),
         "CTCB_LSTM_PARTS": (["auto", "1", "2", "3", "17", "499", "500"], "501"),
         "CTCB_SWEEP_PARTS": (["auto", "1", "2", "3", "17", "499", "500"], "501"),
         "CTCB_STALL": (["off", "main", "side"], "both"),
         "CTCB_STALL_US": (["1", "2", "500", "2000", "99999", "100000"], "100001")}


def _ckpt_refuses():
    """Whether the CTC plan of one 300-frame utterance with 200 labels is refused, as it is under CTCB_CTC=ckpt only
    (the plan query needs no device)."""
    import _ctcb
    out = (ctypes.c_int32 * 8)()
    return _ctcb.lib.ctcb_debug_ctc_plan(1, 300, 20, 200, 256, 256, 6000, 20, out) == -1


def test_set_knob_takes_the_documented_values_only():
    import _ctcb
    lib = _ctcb.lib
    assert lib.ctcb_debug_set_knob(b"CTCB_NO_SUCH_KNOB", b"1") == -1 and b"unknown knob" in lib.ctcb_last_error()
    assert lib.ctcb_debug_set_knob(None, b"1") == -1
    for name, (good, bad) in KNOBS.items():
        for v in good:
            assert lib.ctcb_debug_set_knob(name.encode(), v.encode()) == 0, (name, v, lib.ctcb_last_error())
        for v in (bad, ""):
            assert lib.ctcb_debug_set_knob(name.encode(), v.encode()) == -1, (name, v)
            assert name.encode() in lib.ctcb_last_error()
        assert lib.ctcb_debug_set_knob(name.encode(), None) == 0
    for v in ("0", "01", "-1", "+2", "2x", " 2", "4294967298"):     # the partition count is a plain decimal 1..500
        assert lib.ctcb_debug_set_knob(b"CTCB_LSTM_PARTS", v.encode()) == -1, v
        assert lib.ctcb_debug_set_knob(b"CTCB_SWEEP_PARTS", v.encode()) == -1, v
        assert lib.ctcb_debug_set_knob(b"CTCB_STALL_US", v.encode()) == -1, v     # and the stall 1..100000 us
    for v in ("auto", "off", "main"):                                  # the stall length has no named value
        assert lib.ctcb_debug_set_knob(b"CTCB_STALL_US", v.encode()) == -1, v
    # a refused value leaves the table as it was
    assert lib.ctcb_debug_set_knob(b"CTCB_CTC", b"ckpt") == 0 and _ckpt_refuses()
    assert lib.ctcb_debug_set_knob(b"CTCB_CTC", b"pa") == -1 and _ckpt_refuses()
    assert lib.ctcb_debug_set_knob(b"CTCB_CTC", b"auto") == 0 and not _ckpt_refuses()
    assert lib.ctcb_debug_set_ctc_kernel(4) == 0 and _ckpt_refuses()
    assert lib.ctcb_debug_set_knob(b"CTCB_CTC", None) == 0


def test_set_knob_null_restores_the_environment():
    """The library reads the environment at its first use, so this runs in a fresh process started with CTCB_CTC=ckpt
    (ctypes only, no device): a change overrides it, and NULL brings it back."""
    import subprocess
    import sys
    code = "\n".join([
        "import ctypes, sys",
        "sys.path.insert(0, %r)" % os.path.join(ROOT, "stanford-ctc_b200"),
        "from _ctcb import lib",
        "out = (ctypes.c_int32 * 8)()",
        "refused = lambda: lib.ctcb_debug_ctc_plan(1, 300, 20, 200, 256, 256, 6000, 20, out) == -1",
        "assert refused()",
        "assert lib.ctcb_debug_set_knob(b'CTCB_CTC', b'auto') == 0 and not refused()",
        "assert lib.ctcb_debug_set_knob(b'CTCB_CTC', None) == 0 and refused()"])
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CTCB_CTC="ckpt"), capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]


def test_ctc_workspace_never_shrinks_as_the_batch_grows():
    """A buffer sized once for the largest call (the BRNN sizes its CTC area for maxB) must serve every smaller call:
    the size is monotone in B, Tmax and the label count, and covers two trellis planes for each of the first 256
    utterances (the frame-parallel kernel) and one for every utterance."""
    import _ctcb
    ws = _ctcb.lib.ctcb_ctc_workspace_bytes
    for T, L in ((16, 5), (100, 30), (5000, 300)):
        sizes = [ws(B, T, L) for B in range(1, 1025)]
        assert all(a <= b for a, b in zip(sizes, sizes[1:])), (T, L)
        plane = ws(1, T, L) // 2
        assert all(s >= plane * max(B, 2 * min(B, 256)) for B, s in enumerate(sizes, 1))
    for B in (1, 200, 256, 260, 1000):
        sizes = [ws(B, T, 30) for T in range(1, 400)]
        assert all(a <= b for a, b in zip(sizes, sizes[1:])), B
        sizes = [ws(B, 100, L) for L in range(0, 512)]
        assert all(a <= b for a, b in zip(sizes, sizes[1:])), B
    # the C3-like net of maxB 260, maxT 16, 5 labels: room for a 200-utterance call's 400 planes of 16 x 64 + 2 doubles
    assert ws(260, 16, 5) >= ws(200, 16, 5) == 400 * (16 * 64 + 2) * 8


def test_product_never_imports_the_oracle():
    """The product path must not route through oracle/ (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "stanford-ctc_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in txt.replace("# oracle", ""), "%s mentions the oracle" % f


def test_product_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import numpy as np
    import ctc_fast
    p = np.asfortranarray(np.full((4, 5), 0.25))
    with pytest.raises(RuntimeError):
        ctc_fast.ctc_loss(p, np.array([1, 2], dtype=np.int32))
    with pytest.raises(ValueError):                       # reference contract checked before the device
        ctc_fast.ctc_loss(np.ascontiguousarray(p), np.array([1, 2], dtype=np.int32))
    import nnets.brnnet as rnnet
    with pytest.raises(RuntimeError):
        rnnet.NNet(5, 4, 8, 2, 10, temporalLayer=1)
