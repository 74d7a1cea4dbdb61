"""_ctcb.py -- ctypes binding of libctcb200.so (the C ABI declared in include/ctcb200.h).

PyTorch is used by the callers only as the owner of device memory and streams: every entry point
here takes raw device pointers (`tensor.data_ptr()`), sizes and a `cudaStream_t`.  There is no CPU
fallback: if the shared library is missing this module raises at import time.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctcb200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "libctcb200.so not found at %s -- build it with `make -C %s/csrc` or "
        "`python -c 'import __graft_entry__ as g; g.build()'`; there is no CPU fallback" % (LIB_PATH, _HERE))

lib = ctypes.CDLL(LIB_PATH)

c_int, c_i64, c_f32, c_vp, c_sz = ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t


PART_FIRST, PART_LAST = 1, 2      # CTCB_PART_FIRST / CTCB_PART_LAST (ctcb_brnn_cost_and_grad_part)
CELLS = {"relu": 0, "lstm": 1}   # ctcb_brnn_config.cell


class BrnnConfig(ctypes.Structure):
    _fields_ = [("inputDim", ctypes.c_int32), ("outputDim", ctypes.c_int32), ("layerSize", ctypes.c_int32),
                ("numLayers", ctypes.c_int32), ("temporalLayer", ctypes.c_int32), ("maxT", ctypes.c_int32),
                ("maxB", ctypes.c_int32), ("maxLabels", ctypes.c_int32), ("reg", ctypes.c_float),
                ("maxAct", ctypes.c_float), ("unidirectional", ctypes.c_int32), ("numTemporal", ctypes.c_int32),
                ("cell", ctypes.c_int32), ("layerNorm", ctypes.c_int32), ("subsample", ctypes.c_int32),
                ("subsampleLayer", ctypes.c_int32), ("peephole", ctypes.c_int32), ("maskFeatDim", ctypes.c_int32),
                ("weightNoise", ctypes.c_int32), ("zoneout", ctypes.c_int32), ("interLayer", ctypes.c_int32),
                ("interWeight", ctypes.c_float), ("selfCondition", ctypes.c_int32), ("tf32", ctypes.c_int32)]


_PROTOS = {
    "ctcb_version": (c_int, []),
    "ctcb_last_error": (ctypes.c_char_p, []),
    "ctcb_launch_count": (ctypes.c_uint64, []),
    "ctcb_profile_enable": (None, [c_int]),
    "ctcb_profile_report": (c_int, [ctypes.c_char_p, c_sz]),
    "ctcb_ctc_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "ctcb_ctc_loss_grad_f32": (c_int, [c_vp, c_int, c_i64, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                       c_int, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_ctc_best_path_f32": (c_int, [c_vp, c_i64, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                       c_vp, c_vp]),
    "ctcb_ctc_blankforce_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "ctcb_ctc_blankforce_loss_grad_f32": (c_int, [c_vp, c_int, c_i64, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int,
                                                  c_int, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_gemm_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "ctcb_gemm_f32": (c_int, [c_int, c_int, c_int, c_int, c_int, c_f32, c_vp, c_i64, c_vp, c_i64, c_f32, c_vp,
                              c_i64, c_vp, c_int, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_gemm_pair_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "ctcb_gemm_pair_f32": (c_int, [c_int, c_int, c_int, c_int, c_int, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp, c_i64,
                                   c_f32, c_vp, c_vp, c_i64, c_vp, c_sz, c_vp]),
    "ctcb_debug_gemm_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_i64, c_int,
                                     ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_gemm_tf32": (c_int, [c_int, c_int, c_int, c_int, c_int, c_f32, c_vp, c_i64, c_vp, c_i64, c_f32, c_vp,
                               c_i64, c_vp, c_int, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_gemm_pair_tf32": (c_int, [c_int, c_int, c_int, c_int, c_int, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp, c_i64,
                                    c_f32, c_vp, c_vp, c_i64, c_vp, c_sz, c_vp]),
    "ctcb_debug_gemm_plan_tf32": (c_int, [c_int, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_i64, c_int,
                                          ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_debug_set_knob": (c_int, [ctypes.c_char_p, ctypes.c_char_p]),
    "ctcb_debug_gemm_trace": (c_int, [c_vp]),
    "ctcb_debug_set_ctc_kernel": (c_int, [c_int]),
    "ctcb_debug_ctc_plan": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_i64, c_i64,
                                    ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_brnn_param_count": (c_i64, [ctypes.POINTER(BrnnConfig)]),
    "ctcb_brnn_num_tensors": (c_int, [ctypes.POINTER(BrnnConfig)]),
    "ctcb_brnn_tensor_info": (c_int, [ctypes.POINTER(BrnnConfig), c_int, ctypes.POINTER(c_i64),
                                      ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_brnn_workspace_bytes": (c_sz, [ctypes.POINTER(BrnnConfig)]),
    "ctcb_brnn_error_flag_offset": (c_sz, [ctypes.POINTER(BrnnConfig)]),
    "ctcb_brnn_forward_workspace_bytes": (c_sz, [ctypes.POINTER(BrnnConfig), ctypes.POINTER(c_sz)]),
    "ctcb_brnn_activation_offset": (c_int, [ctypes.POINTER(BrnnConfig), c_int, c_int, ctypes.POINTER(c_sz),
                                            ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_brnn_create": (c_int, [ctypes.POINTER(BrnnConfig), ctypes.POINTER(c_vp)]),
    "ctcb_brnn_destroy": (None, [c_vp]),
    "ctcb_brnn_cost_and_grad": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                        c_vp, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_brnn_cost_and_grad_part": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp,
                                             c_vp, c_vp, c_vp, c_int, c_vp, c_sz, c_vp]),
    "ctcb_brnn_sweep_f32": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32,
                                    c_vp, c_sz, c_vp]),
    "ctcb_brnn_sweep_tf32": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                     c_f32, c_vp, c_sz, c_vp]),
    "ctcb_brnn_sweep_workspace_bytes": (c_sz, [c_int, c_int]),
    "ctcb_sweep_uses_tensor_cores": (c_int, [c_int, c_int]),
    "ctcb_lstm_sweep_workspace_bytes": (c_sz, [c_int, c_int]),
    "ctcb_lstm_sweep_f32": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                    c_vp, c_vp, c_sz, c_vp]),
    "ctcb_lstm_sweep_peephole_f32": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                             c_vp, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "ctcb_lstm_peephole_grad_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int]),
    "ctcb_lstm_peephole_grad_f32": (c_int, [c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_sz, c_vp]),
    "ctcb_debug_lstm_plan": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_debug_lstm_zoneout_plan": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_lstm_sweep_zoneout_workspace_bytes": (c_sz, [c_int, c_int]),
    "ctcb_lstm_sweep_zoneout_f32": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                            c_vp, c_vp, c_vp, c_vp, c_f32, c_f32, c_int, ctypes.c_uint64, c_vp, c_i64,
                                            c_i64, c_int, c_vp, c_sz, c_vp]),
    "ctcb_brnn_set_zoneout": (c_int, [c_vp, c_f32, c_f32, ctypes.c_uint64, c_vp]),
    "ctcb_layernorm_workspace_bytes": (c_sz, [c_i64, c_int]),
    "ctcb_layernorm_forward_f32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_vp]),
    "ctcb_layernorm_backward_f32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_sz,
                                            c_vp]),
    "ctcb_colsum_workspace_bytes": (c_sz, [c_i64, c_int]),
    "ctcb_colsum_f32": (c_int, [c_vp, c_i64, c_int, c_vp, c_int, c_vp, c_sz, c_vp]),
    "ctcb_debug_colsum_plan": (c_int, [c_i64, c_int, c_vp, ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_softmax_rows_f32": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp]),
    "ctcb_softmax_rows_backward_f32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_vp]),
    "ctcb_frame_stack_f32": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "ctcb_frame_unstack_f32": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "ctcb_debug_sweep_plan": (c_int, [c_int, c_int, c_int, ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_debug_sweep_plan_tf32": (c_int, [c_int, c_int, c_int, ctypes.POINTER(ctypes.c_int32)]),
    "ctcb_brnn_set_deferred_l2": (c_int, [c_vp, c_int]),
    "ctcb_brnn_apply_l2_f32": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "ctcb_brnn_set_dropout": (c_int, [c_vp, c_f32, ctypes.c_uint64, c_vp]),
    "ctcb_brnn_set_dropout_utts": (c_int, [c_vp, c_i64, c_i64]),
    "ctcb_dropout_advance": (c_int, [c_vp, c_vp]),
    "ctcb_brnn_set_input_masks": (c_int, [c_vp, c_int, c_int, c_int, c_int, ctypes.c_double, ctypes.c_uint64, c_vp]),
    "ctcb_input_mask_f32": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, ctypes.c_double,
                                    ctypes.c_uint64, c_vp, c_i64, c_i64, c_vp, c_vp]),
    "ctcb_brnn_set_weight_noise": (c_int, [c_vp, c_f32, ctypes.c_uint64, c_vp]),
    "ctcb_brnn_weight_noise_f32": (c_int, [c_vp, c_vp, c_vp, c_vp]),
    "ctcb_comm_get_unique_id": (c_int, [c_vp]),
    "ctcb_comm_create": (c_int, [c_vp, c_int, c_int, ctypes.POINTER(c_vp)]),
    "ctcb_comm_destroy": (None, [c_vp]),
    "ctcb_comm_rank": (c_int, [c_vp]),
    "ctcb_comm_world": (c_int, [c_vp]),
    "ctcb_allreduce_grads": (c_int, [c_vp, c_vp, c_i64, c_vp]),
    "ctcb_brnn_set_comm": (c_int, [c_vp, c_vp]),
    "ctcb_brnn_exchange_only": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "ctcb_graph_capture_begin": (c_int, [c_vp]),
    "ctcb_graph_capture_end": (c_int, [c_vp, ctypes.POINTER(c_vp)]),
    "ctcb_graph_launch": (c_int, [c_vp, c_vp]),
    "ctcb_graph_destroy": (None, [c_vp]),
    "ctcb_axpy_f32": (c_int, [c_vp, c_vp, c_f32, c_i64, c_vp]),
    "ctcb_sumsq_f32": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp]),
    "ctcb_sgd_nesterov_step_f32": (c_int, [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_vp, c_vp, c_vp]),
    "ctcb_adagrad_step_f32": (c_int, [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "ctcb_adam_step_f32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp, c_vp, c_vp,
                                   c_vp]),
    "ctcb_ema_update_f32": (c_int, [c_vp, c_vp, c_i64, c_f32, c_vp, c_vp, c_vp]),
}

EXPORTS = sorted(_PROTOS)

for _name, (_res, _args) in _PROTOS.items():
    _fn = getattr(lib, _name)          # AttributeError here == header/library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


class CtcbError(RuntimeError):
    pass


def check(rc):
    """Turn a negative status code into the Python exception the reference surface would raise."""
    if rc == 0:
        return
    msg = lib.ctcb_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    if rc == -3:
        raise MemoryError(msg)
    raise CtcbError("libctcb200 error %d: %s" % (rc, msg))


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("stanford-ctc_b200 needs a CUDA device (H100, sm_90a); no CPU fallback exists")
    return torch
