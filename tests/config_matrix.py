"""config_matrix.py -- TEST INFRASTRUCTURE ONLY: every config-level answer of libctcb200 over a matrix of nets, reduced
to one 64-bit digest per config.

The queries are the ones a caller sizes and lays out a net with: ctcb_brnn_param_count, ctcb_brnn_num_tensors,
ctcb_brnn_tensor_info of every index and one out of range on each side, both workspace sizes with the error-flag
offsets, ctcb_brnn_activation_offset for what 0..6 and layers 0..numLayers+2 (return code, offset, width) and the return
code of ctcb_brnn_create (clipped-ReLU nets only: an LSTM net's create asks the device whether its sweep fits).
tests/golden/subsample_configs.npz (no device visible) and subsample_configs_h100_sxm.npz (an H100 SXM: sm_90, 132
SMs) hold the digests of the build before frame subsampling existed; some answers depend on the device the contraction
and sweep planners see, hence one file per kind of machine.  tests/test_subsample_cpu.py checks that subsample = 0 and
1 still give them, and tests/golden/gen_subsample_golden.py writes them from a given build of the library."""
import ctypes
import hashlib
import itertools

import numpy as np

# (D, K, H, N, tl, nt, uni, cell, ln, (T, B)): 2 * 2 * 5 * 4 * 5 * 2 * 2 * 2 * 2 * 4 = 25,600 configs, invalid ones
# (tl beyond N, stacks that do not fit) included
MATRIX = list(itertools.product((13, 41), (11, 62), (64, 70, 512, 1024, 1824), (1, 2, 3, 5), (-1, 0, 1, 2, 3), (0, 2),
                                (0, 1), (0, 1), (0, 1), ((1, 1), (37, 5), (200, 32), (800, 128))))


def bind(lib, BrnnConfig):
    """Prototypes of the queries on `lib` (any build of libctcb200.so)."""
    P = ctypes.POINTER(BrnnConfig)
    c_sz, c_i64, c_i32 = ctypes.c_size_t, ctypes.c_int64, ctypes.c_int32
    protos = {
        "ctcb_brnn_param_count": (c_i64, [P]), "ctcb_brnn_num_tensors": (ctypes.c_int, [P]),
        "ctcb_brnn_tensor_info": (ctypes.c_int, [P, ctypes.c_int, ctypes.POINTER(c_i64), ctypes.POINTER(c_i32),
                                                 ctypes.POINTER(c_i32)]),
        "ctcb_brnn_workspace_bytes": (c_sz, [P]), "ctcb_brnn_error_flag_offset": (c_sz, [P]),
        "ctcb_brnn_forward_workspace_bytes": (c_sz, [P, ctypes.POINTER(c_sz)]),
        "ctcb_brnn_activation_offset": (ctypes.c_int, [P, ctypes.c_int, ctypes.c_int, ctypes.POINTER(c_sz),
                                                       ctypes.POINTER(c_i32)]),
        "ctcb_brnn_create": (ctypes.c_int, [P, ctypes.POINTER(ctypes.c_void_p)]),
        "ctcb_brnn_destroy": (None, [ctypes.c_void_p]),
    }
    for name, (res, args) in protos.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def answers(lib, cfg):
    """Every answer for one config, as a list of ints."""
    r = ctypes.byref(cfg)
    out = [lib.ctcb_brnn_param_count(r)]
    n = lib.ctcb_brnn_num_tensors(r)
    out.append(n)
    off, rows, cols = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
    for idx in range(-1, n + 1):
        off.value = rows.value = cols.value = -7
        rc = lib.ctcb_brnn_tensor_info(r, idx, ctypes.byref(off), ctypes.byref(rows), ctypes.byref(cols))
        out += [rc, off.value, rows.value, cols.value] if rc == 0 else [rc]
    out += [lib.ctcb_brnn_workspace_bytes(r), lib.ctcb_brnn_error_flag_offset(r)]
    f = ctypes.c_size_t(12345)
    out += [lib.ctcb_brnn_forward_workspace_bytes(r, ctypes.byref(f)), f.value]
    o, w = ctypes.c_size_t(), ctypes.c_int32()
    for what in range(7):
        for layer in range(0, cfg.numLayers + 3):
            o.value, w.value = 1, -7
            rc = lib.ctcb_brnn_activation_offset(r, what, layer, ctypes.byref(o), ctypes.byref(w))
            out += [rc, o.value, w.value] if rc == 0 else [rc]
    if cfg.cell == 0:
        h = ctypes.c_void_p()
        rc = lib.ctcb_brnn_create(r, ctypes.byref(h))
        out.append(rc)
        if rc == 0:
            lib.ctcb_brnn_destroy(h)
    return out


def config(BrnnConfig, entry, subsample=0, subsampleLayer=0):
    D, K, H, N, tl, nt, uni, cell, ln, (T, B) = entry
    cfg = BrnnConfig(D, K, H, N, tl, T, B, 20, 0.0, 20.0, uni, nt, cell, ln)
    if hasattr(cfg, "subsample"):
        cfg.subsample, cfg.subsampleLayer = subsample, subsampleLayer
    return cfg


def digest(values):
    return int.from_bytes(hashlib.sha256(np.asarray(values, dtype=np.int64).tobytes()).digest()[:8], "little",
                          signed=True)
