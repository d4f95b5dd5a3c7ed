"""ctypes binding of libb2cnn.so (include/b2cnn.h) -- the only way Python reaches the kernels.

This is the binding a maintainer of the reference would add beside bin/models.py to replace
``model(x, age)`` (bin/predictStream.py:157); INTEGRATION.md shows it in isolation.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2CNN_LIB: load another build of the same library (e.g. an instrumented copy)
_LIB_PATH = os.environ.get("B2CNN_LIB") or os.path.join(_HERE, "lib", "libb2cnn.so")

OK, EINVAL, EARCH, EVIEW, ECUDA, ESTATE = range(6)
DTYPE_F32, DTYPE_BF16 = 0, 1
MODE_INDEPENDENT, MODE_SEQUENCE = 0, 1
TRAIN_FROZEN_CONV = 1          # b2cnn_train_backward_ex flag (include/b2cnn.h)
PATH_AUTO, PATH_GENERIC, PATH_TENSORCORE = 0, 1, 2
FLAG_AFFINE = 1
SAMPLES_ADC16, SAMPLES_F64, SAMPLES_GRID = 0, 1, 2

# every symbol include/b2cnn.h declares (tests/test_host.py::test_library_exports_every_declared_symbol checks the list)
SYMBOLS = ("b2cnn_l_out", "b2cnn_weight_count", "b2cnn_create", "b2cnn_destroy",
           "b2cnn_set_weights", "b2cnn_workspace_bytes", "b2cnn_workspace_bytes_for", "b2cnn_forward", "b2cnn_forward_pitched", "b2cnn_forward_host",
           "b2cnn_features", "b2cnn_set_option", "b2cnn_get_option", "b2cnn_last_launch_count",
           "b2cnn_last_path", "b2cnn_last_stage_ms", "b2cnn_last_error", "b2cnn_version", "b2cnn_train_workspace_bytes", "b2cnn_train_step",
           "b2cnn_train_step_weighted", "b2cnn_train_forward", "b2cnn_train_backward", "b2cnn_train_backward_ex",
           "b2cnn_train_workspace_bytes_seq", "b2cnn_train_step_seq", "b2cnn_train_forward_seq", "b2cnn_train_backward_seq",
           "b2cnn_workspace_bytes_seq", "b2cnn_forward_seq",
           "b2cnn_train_workspace_bytes_record", "b2cnn_train_step_record", "b2cnn_train_forward_record", "b2cnn_train_backward_record",
           "b2cnn_prep_window_count", "b2cnn_prep_workspace_bytes", "b2cnn_prep_windows",
           "b2cnn_ring_create", "b2cnn_ring_destroy", "b2cnn_ring_reset", "b2cnn_ring_set_signals", "b2cnn_ring_push",
           "b2cnn_slide_create", "b2cnn_slide_destroy", "b2cnn_slide_reset", "b2cnn_slide_push", "b2cnn_slide_features",
           "b2cnn_slide_admit_workspace_bytes", "b2cnn_slide_admit", "b2cnn_slide_discharge", "b2cnn_slide_samples_seen",
           "b2cnn_slide_create_path", "b2cnn_slide_path",
           "b2cnn_slide_describe_state", "b2cnn_slide_state_workspace_bytes", "b2cnn_slide_export", "b2cnn_slide_import",
           "b2cnn_slide_set_heads", "b2cnn_slide_set_heads_ex", "b2cnn_slide_n_heads", "b2cnn_slide_push_heads",
           "b2cnn_slide_create_ex", "b2cnn_slide_mode", "b2cnn_slide_export_ex", "b2cnn_slide_import_ex",
           "b2cnn_record_workspace_bytes", "b2cnn_score_record", "b2cnn_record_workspace_bytes_ex", "b2cnn_score_record_ex",
           "b2cnn_score_record_state", "b2cnn_slide_admit_ex", "b2cnn_train_step_record_state", "b2cnn_train_forward_record_state",
           "b2cnn_train_backward_record_state", "b2cnn_record_workspace_bytes_heads", "b2cnn_score_record_heads",
           "b2cnn_train_heads_workspace_bytes", "b2cnn_train_heads_step", "b2cnn_train_heads_workspace_bytes_record",
           "b2cnn_train_heads_step_record",
           "b2cnn_decode_sample_messages", "b2cnn_decode_array_messages", "b2cnn_parse_decimal", "b2cnn_frame_check")


class LibraryNotBuilt(RuntimeError):
    pass


class Config(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in
                ("in_channels", "k1", "c_mid", "k2", "pool_k", "pool_s", "hidden", "layers",
                 "window", "lstm_input", "act", "flags")] + \
               [("age_coef", ctypes.c_float), ("device", ctypes.c_int32)]


class FrameHeader(ctypes.Structure):
    """b2cnn_frame_header: one binary frame per trigger for all patients (include/b2cnn.h)."""
    _fields_ = [("magic", ctypes.c_uint32), ("version", ctypes.c_uint16), ("kind", ctypes.c_uint16), ("n_patients", ctypes.c_uint32),
                ("n_new", ctypes.c_uint32), ("n_sig", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("first_index", ctypes.c_uint64)]


FRAME_MAGIC = 0x46573242


class SlideStateHeader(ctypes.Structure):
    """b2cnn_slide_state_header: what a SlidingScorer's exported patients fit (include/b2cnn.h)."""
    _fields_ = [("magic", ctypes.c_uint32), ("version", ctypes.c_uint16), ("path", ctypes.c_uint16), ("dtype", ctypes.c_int32),
                ("in_channels", ctypes.c_int32), ("window", ctypes.c_int32), ("lstm_input", ctypes.c_int32),
                ("feature_stride", ctypes.c_int32), ("tail_len", ctypes.c_int32), ("frontend_digest", ctypes.c_uint64)]


SLIDE_STATE_MAGIC, SLIDE_STATE_VERSION = 0x53533242, 1
SLIDE_MAX_HEADS = 8                  # B2CNN_SLIDE_MAX_HEADS
SLIDE_HEADS_SHORTER_WINDOWS = 1      # B2CNN_SLIDE_HEADS_SHORTER_WINDOWS


class Adam(ctypes.Structure):
    """b2cnn_adam (include/b2cnn.h): torch.optim.Adam hyper-parameters."""
    _fields_ = [("lr", ctypes.c_float), ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("eps", ctypes.c_float)]


class PrepConfig(ctypes.Structure):
    """b2cnn_prep_config: the reference's window constants (config.cfg, processStream.py:199, predictStream.py:252)."""
    _fields_ = [(n, ctypes.c_int32) for n in ("n_channels", "window_points", "grid_s", "smooth_s", "stride_s")]


_lib: Optional[ctypes.CDLL] = None


def lib_path() -> str:
    return _LIB_PATH


def load_library() -> ctypes.CDLL:
    """Load libb2cnn.so; raises LibraryNotBuilt (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise LibraryNotBuilt(
            f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  There is no CPU fallback for this path.")
    lib = ctypes.CDLL(_LIB_PATH)
    c_i64, c_int, c_vp = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p
    cfgp = ctypes.POINTER(Config)
    lib.b2cnn_l_out.argtypes = [cfgp]; lib.b2cnn_l_out.restype = c_i64
    lib.b2cnn_weight_count.argtypes = [cfgp]; lib.b2cnn_weight_count.restype = c_i64
    lib.b2cnn_create.argtypes = [cfgp, ctypes.POINTER(c_vp)]; lib.b2cnn_create.restype = c_int
    lib.b2cnn_destroy.argtypes = [c_vp]; lib.b2cnn_destroy.restype = None
    lib.b2cnn_set_weights.argtypes = [c_vp, c_vp, c_i64, c_int, c_vp]; lib.b2cnn_set_weights.restype = c_int
    lib.b2cnn_workspace_bytes.argtypes = [c_vp, c_i64, c_int]; lib.b2cnn_workspace_bytes.restype = c_i64
    lib.b2cnn_workspace_bytes_for.argtypes = [c_vp, c_i64, c_int, c_int]; lib.b2cnn_workspace_bytes_for.restype = c_i64
    lib.b2cnn_forward.argtypes = [c_vp, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_forward.restype = c_int
    lib.b2cnn_forward_pitched.argtypes = [c_vp, c_vp, c_int, c_i64, c_i64, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_forward_pitched.restype = c_int
    lib.b2cnn_forward_host.argtypes = [c_vp, c_vp, c_int, c_i64, c_vp, c_i64, c_int, c_int, c_vp]
    lib.b2cnn_forward_host.restype = c_int
    lib.b2cnn_features.argtypes = [c_vp, c_vp, c_int, c_i64, c_vp, c_vp]; lib.b2cnn_features.restype = c_int
    lib.b2cnn_set_option.argtypes = [c_vp, ctypes.c_char_p, c_i64]; lib.b2cnn_set_option.restype = c_int
    lib.b2cnn_get_option.argtypes = [c_vp, ctypes.c_char_p]; lib.b2cnn_get_option.restype = c_i64
    lib.b2cnn_last_launch_count.argtypes = [c_vp]; lib.b2cnn_last_launch_count.restype = c_i64
    lib.b2cnn_last_path.argtypes = [c_vp]; lib.b2cnn_last_path.restype = c_int
    lib.b2cnn_last_stage_ms.argtypes = [c_vp, c_int]; lib.b2cnn_last_stage_ms.restype = ctypes.c_double
    pcfg = ctypes.POINTER(PrepConfig)
    lib.b2cnn_prep_window_count.argtypes = [c_i64, ctypes.c_double, pcfg]; lib.b2cnn_prep_window_count.restype = c_i64
    lib.b2cnn_prep_workspace_bytes.argtypes = [c_i64, ctypes.c_double, ctypes.c_int32, pcfg]
    lib.b2cnn_prep_workspace_bytes.restype = c_i64
    lib.b2cnn_prep_windows.argtypes = [c_vp, c_i64, ctypes.c_int32, c_vp, ctypes.c_int32, c_vp, c_vp, ctypes.c_double, pcfg,
                                       c_vp, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_prep_windows.restype = c_int
    c_i32 = ctypes.c_int32
    lib.b2cnn_ring_create.argtypes = [pcfg, c_i32, c_i32, ctypes.c_double, c_i32, ctypes.POINTER(c_vp)]; lib.b2cnn_ring_create.restype = c_int
    lib.b2cnn_ring_destroy.argtypes = [c_vp]; lib.b2cnn_ring_destroy.restype = None
    lib.b2cnn_ring_reset.argtypes = [c_vp, c_vp]; lib.b2cnn_ring_reset.restype = c_int
    lib.b2cnn_ring_set_signals.argtypes = [c_vp, c_i32, c_vp, c_i32, c_vp, c_vp, c_vp]; lib.b2cnn_ring_set_signals.restype = c_int
    lib.b2cnn_ring_push.argtypes = [c_vp, c_vp, c_int, c_i64, c_vp, c_int, ctypes.POINTER(c_i32), ctypes.POINTER(c_i64),
                                    ctypes.POINTER(ctypes.c_double), c_vp]
    lib.b2cnn_ring_push.restype = c_int
    lib.b2cnn_slide_create.argtypes = [c_vp, c_i32, c_i32, c_int, ctypes.POINTER(c_vp)]; lib.b2cnn_slide_create.restype = c_int
    lib.b2cnn_slide_destroy.argtypes = [c_vp]; lib.b2cnn_slide_destroy.restype = None
    lib.b2cnn_slide_reset.argtypes = [c_vp, c_vp]; lib.b2cnn_slide_reset.restype = c_int
    lib.b2cnn_slide_push.argtypes = [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, ctypes.POINTER(c_i32), ctypes.POINTER(c_i64), c_vp]
    lib.b2cnn_slide_push.restype = c_int
    lib.b2cnn_slide_features.argtypes = [c_vp, c_vp, c_vp]; lib.b2cnn_slide_features.restype = c_int
    lib.b2cnn_slide_admit_workspace_bytes.argtypes = [c_vp, c_i32, c_i64]; lib.b2cnn_slide_admit_workspace_bytes.restype = c_i64
    lib.b2cnn_slide_admit.argtypes = [c_vp, c_vp, c_i32, c_vp, c_i64, c_i64, c_int, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_admit.restype = c_int
    lib.b2cnn_slide_discharge.argtypes = [c_vp, c_vp, c_i32, c_vp]; lib.b2cnn_slide_discharge.restype = c_int
    lib.b2cnn_slide_samples_seen.argtypes = [c_vp, c_vp, c_vp]; lib.b2cnn_slide_samples_seen.restype = c_int
    lib.b2cnn_slide_create_path.argtypes = [c_vp, c_i32, c_i32, c_int, c_int, ctypes.POINTER(c_vp)]
    lib.b2cnn_slide_create_path.restype = c_int
    lib.b2cnn_slide_path.argtypes = [c_vp]; lib.b2cnn_slide_path.restype = c_int
    hdrp = ctypes.POINTER(SlideStateHeader)
    lib.b2cnn_slide_describe_state.argtypes = [c_vp, hdrp]; lib.b2cnn_slide_describe_state.restype = c_int
    lib.b2cnn_slide_state_workspace_bytes.argtypes = [c_vp, c_i32]; lib.b2cnn_slide_state_workspace_bytes.restype = c_i64
    lib.b2cnn_slide_export.argtypes = [c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, hdrp, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_export.restype = c_int
    lib.b2cnn_slide_import.argtypes = [c_vp, c_vp, c_i32, hdrp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_import.restype = c_int
    lib.b2cnn_slide_set_heads.argtypes = [c_vp, c_vp, c_i32, c_vp]; lib.b2cnn_slide_set_heads.restype = c_int
    lib.b2cnn_slide_set_heads_ex.argtypes = [c_vp, c_vp, c_i32, c_i32, c_vp]; lib.b2cnn_slide_set_heads_ex.restype = c_int
    lib.b2cnn_slide_n_heads.argtypes = [c_vp]; lib.b2cnn_slide_n_heads.restype = c_int
    lib.b2cnn_slide_push_heads.argtypes = lib.b2cnn_slide_push.argtypes; lib.b2cnn_slide_push_heads.restype = c_int
    lib.b2cnn_slide_create_ex.argtypes = [c_vp, c_i32, c_i32, c_int, c_int, c_int, ctypes.POINTER(c_vp)]
    lib.b2cnn_slide_create_ex.restype = c_int
    lib.b2cnn_slide_mode.argtypes = [c_vp]; lib.b2cnn_slide_mode.restype = c_int
    lib.b2cnn_slide_export_ex.argtypes = [c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, hdrp, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_export_ex.restype = c_int
    lib.b2cnn_slide_import_ex.argtypes = [c_vp, c_vp, c_i32, hdrp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_import_ex.restype = c_int
    lib.b2cnn_record_workspace_bytes.argtypes = [c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_int]
    lib.b2cnn_record_workspace_bytes.restype = c_i64
    lib.b2cnn_score_record.argtypes = [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_i64, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_score_record.restype = c_int
    lib.b2cnn_record_workspace_bytes_ex.argtypes = [c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int]
    lib.b2cnn_record_workspace_bytes_ex.restype = c_i64
    lib.b2cnn_score_record_ex.argtypes = [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_vp, c_i64, c_int, c_vp, c_vp,
                                          c_i64, c_vp]
    lib.b2cnn_score_record_ex.restype = c_int
    lib.b2cnn_score_record_state.argtypes = [c_vp, c_vp, c_int, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_vp, c_i64, c_int, c_vp, c_vp,
                                             c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_score_record_state.restype = c_int
    lib.b2cnn_record_workspace_bytes_heads.argtypes = [c_vp, c_i32, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int]
    lib.b2cnn_record_workspace_bytes_heads.restype = c_i64
    lib.b2cnn_score_record_heads.argtypes = [c_vp, c_vp, c_i32, c_vp, c_int, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_vp, c_i64, c_int,
                                             c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_score_record_heads.restype = c_int
    lib.b2cnn_slide_admit_ex.argtypes = [c_vp, c_vp, c_i32, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_slide_admit_ex.restype = c_int
    lib.b2cnn_decode_sample_messages.argtypes = [c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_vp]
    lib.b2cnn_decode_sample_messages.restype = c_int
    lib.b2cnn_decode_array_messages.argtypes = [c_vp, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp]
    lib.b2cnn_decode_array_messages.restype = c_int
    lib.b2cnn_parse_decimal.argtypes = [ctypes.c_char_p, c_i64, ctypes.POINTER(c_i32)]; lib.b2cnn_parse_decimal.restype = ctypes.c_double
    lib.b2cnn_frame_check.argtypes = [c_vp, c_i64, ctypes.POINTER(FrameHeader), ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    lib.b2cnn_frame_check.restype = c_int
    lib.b2cnn_train_workspace_bytes.argtypes = [cfgp, c_i64]; lib.b2cnn_train_workspace_bytes.restype = c_i64
    lib.b2cnn_train_step.argtypes = [cfgp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64, c_vp, c_vp, c_int,
                                     c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_step.restype = c_int
    lib.b2cnn_train_step_weighted.argtypes = [cfgp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64, c_vp, c_vp,
                                              ctypes.c_float, c_int, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_step_weighted.restype = c_int
    lib.b2cnn_train_forward.argtypes = [cfgp, c_vp, c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_forward.restype = c_int
    lib.b2cnn_train_backward.argtypes = [cfgp, c_vp, c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_backward.restype = c_int
    lib.b2cnn_train_backward_ex.argtypes = [cfgp, c_vp, c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_i64, c_vp]
    lib.b2cnn_train_backward_ex.restype = c_int
    lib.b2cnn_train_workspace_bytes_seq.argtypes = [cfgp, c_i64, c_vp, c_i64]; lib.b2cnn_train_workspace_bytes_seq.restype = c_i64
    lib.b2cnn_train_step_seq.argtypes = [cfgp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64, c_vp, c_vp,
                                         c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_step_seq.restype = c_int
    lib.b2cnn_train_forward_seq.argtypes = [cfgp, c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_forward_seq.restype = c_int
    lib.b2cnn_train_backward_seq.argtypes = [cfgp, c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_vp,
                                             c_i64, c_vp]
    lib.b2cnn_train_backward_seq.restype = c_int
    lib.b2cnn_train_workspace_bytes_record.argtypes = [cfgp, c_i64, c_i64, c_i64, c_vp, c_int]
    lib.b2cnn_train_workspace_bytes_record.restype = c_i64
    lib.b2cnn_train_step_record.argtypes = [cfgp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64, c_i64, c_i64, c_vp,
                                            c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_step_record.restype = c_int
    lib.b2cnn_train_forward_record.argtypes = [cfgp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_forward_record.restype = c_int
    lib.b2cnn_train_backward_record.argtypes = [cfgp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                c_int, c_vp, c_i64, c_vp]
    lib.b2cnn_train_backward_record.restype = c_int
    lib.b2cnn_train_step_record_state.argtypes = [cfgp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64, c_i64, c_i64,
                                                  c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_step_record_state.restype = c_int
    lib.b2cnn_train_forward_record_state.argtypes = [cfgp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                     c_vp, c_i64, c_vp]
    lib.b2cnn_train_forward_record_state.restype = c_int
    lib.b2cnn_train_backward_record_state.argtypes = [cfgp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                      c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_i64, c_vp]
    lib.b2cnn_train_backward_record_state.restype = c_int
    lib.b2cnn_train_heads_workspace_bytes.argtypes = [cfgp, c_i32, c_i64, c_vp, c_i64]
    lib.b2cnn_train_heads_workspace_bytes.restype = c_i64
    lib.b2cnn_train_heads_step.argtypes = [cfgp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp, c_i64,
                                           c_vp, c_vp, c_vp, c_int, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_heads_step.restype = c_int
    lib.b2cnn_train_heads_workspace_bytes_record.argtypes = [cfgp, c_i32, c_i64, c_i64, c_i64, c_vp, c_int]
    lib.b2cnn_train_heads_workspace_bytes_record.restype = c_i64
    lib.b2cnn_train_heads_step_record.argtypes = [cfgp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.POINTER(Adam), c_int, c_vp,
                                                  c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_train_heads_step_record.restype = c_int
    lib.b2cnn_workspace_bytes_seq.argtypes = [c_vp, c_i64, c_vp, c_i64]; lib.b2cnn_workspace_bytes_seq.restype = c_i64
    lib.b2cnn_forward_seq.argtypes = [c_vp, c_vp, c_int, c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_i64, c_vp]
    lib.b2cnn_forward_seq.restype = c_int
    lib.b2cnn_last_error.argtypes = []; lib.b2cnn_last_error.restype = ctypes.c_char_p
    lib.b2cnn_version.argtypes = []; lib.b2cnn_version.restype = ctypes.c_char_p
    _lib = lib
    return lib


def last_error() -> str:
    return load_library().b2cnn_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    """The reference raises RuntimeError on shape mismatches; so does the drop-in."""
    if rc != OK:
        raise RuntimeError(f"{what}: {last_error()} (b2cnn error {rc})")


def seq_lengths_array(seq_lengths, B: int):
    """``seq_lengths`` (a list, tuple or integer tensor of N >= 1 lengths, each >= 1, adding up to B) as the host int64
    array the ``_seq`` entry points take; ValueError for anything else.  Sequence s is rows o_s .. o_s + n_s - 1 of the
    batch, o_s = n_0 + ... + n_{s-1}."""
    import operator

    import torch
    if isinstance(seq_lengths, (list, tuple)):
        vals = list(seq_lengths)
    elif torch.is_tensor(seq_lengths):
        if seq_lengths.dim() != 1 or seq_lengths.dtype.is_floating_point or seq_lengths.dtype.is_complex \
                or seq_lengths.dtype == torch.bool:
            raise ValueError(f"seq_lengths must be a 1-d integer tensor, got {seq_lengths.dtype} of shape {tuple(seq_lengths.shape)}")
        vals = seq_lengths.tolist()
    else:
        raise ValueError(f"seq_lengths must be a list, tuple or integer tensor, got {type(seq_lengths).__name__}")
    if not vals:
        raise ValueError("seq_lengths must hold at least one sequence")
    out = []
    for i, v in enumerate(vals):
        if isinstance(v, bool):
            raise ValueError(f"seq_lengths[{i}] must be an integer, got bool")
        try:
            v = operator.index(v)
        except TypeError:
            raise ValueError(f"seq_lengths[{i}] must be an integer, got {type(v).__name__}") from None
        if v < 1:
            raise ValueError(f"seq_lengths[{i}] = {v}: every sequence needs at least one window")
        out.append(v)
    if sum(out) != B:
        raise ValueError(f"seq_lengths add up to {sum(out)}, the batch has {B} windows")
    return (ctypes.c_int64 * len(out))(*out)


def record_window_count(N: int, W: int, stride: int) -> int:
    """n_w: the windows of W samples every ``stride`` samples that fit in N samples, (N - W) // stride + 1 (0 when N < W)."""
    return (N - W) // stride + 1 if N >= W else 0


def window_counts_array(window_counts, B: int, N: int, W: int, stride: int):
    """``window_counts`` (None for every recording's n_w windows; else a list, tuple or 1-d integer tensor of B counts,
    each in [0, n_w], adding up to at least 1) as the host int64 array the ``_record`` training calls take, and their sum
    M; ValueError for anything else.  Recording b contributes its windows 0 .. count_b - 1."""
    import operator

    import torch
    n_w = record_window_count(N, W, stride)
    if window_counts is None:
        vals = [n_w] * B
    elif isinstance(window_counts, (list, tuple)):
        vals = list(window_counts)
    elif torch.is_tensor(window_counts):
        if window_counts.dim() != 1 or window_counts.dtype.is_floating_point or window_counts.dtype.is_complex \
                or window_counts.dtype == torch.bool:
            raise ValueError(f"window_counts must be a 1-d integer tensor, got {window_counts.dtype} of shape {tuple(window_counts.shape)}")
        vals = window_counts.tolist()
    else:
        raise ValueError(f"window_counts must be a list, tuple or integer tensor, got {type(window_counts).__name__}")
    if len(vals) != B:
        raise ValueError(f"window_counts has {len(vals)} entries, the batch has {B} recordings")
    out = []
    for i, v in enumerate(vals):
        if isinstance(v, bool):
            raise ValueError(f"window_counts[{i}] must be an integer, got bool")
        try:
            v = operator.index(v)
        except TypeError:
            raise ValueError(f"window_counts[{i}] must be an integer, got {type(v).__name__}") from None
        if not 0 <= v <= n_w:
            raise ValueError(f"window_counts[{i}] = {v}: a recording of N = {N} samples holds 0 .. {n_w} windows of W = {W} "
                             f"every {stride} samples")
        out.append(v)
    if sum(out) < 1:
        raise ValueError(f"the recordings hold no window (N = {N}, W = {W}, stride = {stride}, counts add up to 0)")
    return (ctypes.c_int64 * B)(*out), sum(out)


def make_config(arch, device: int = -1) -> Config:
    return Config(arch.in_channels, arch.k1, arch.c_mid, arch.k2, arch.pool_k, arch.pool_s,
                  arch.hidden, arch.layers, arch.window, arch.l_out, arch.act_id,
                  FLAG_AFFINE if arch.affine else 0, float(arch.age_coef), device)
