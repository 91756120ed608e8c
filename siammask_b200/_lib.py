"""ctypes binding of the C ABI declared in include/siammask_b200.h.

The shared library is the product: if it is missing this module raises — there is no Python or
CPU fallback for any compute entry point."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsiammask_b200.so")

SM_PRECISION_EXACT, SM_PRECISION_FAST = 0, 1
SM_BACKEND_TENSOR, SM_BACKEND_SIMT = 0, 1
SM_TRACK_MASK_FEATURES, SM_TRACK_MASK_HEAD = 1, 2


class SmConfig(C.Structure):
    _fields_ = [("search_size", C.c_int32), ("max_batch", C.c_int32), ("num_slots", C.c_int32),
                ("precision", C.c_int32), ("backend", C.c_int32), ("anchor_num", C.c_int32),
                ("with_mask", C.c_int32)]


class SmTensorDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * 4)]


class SmStepIO(C.Structure):
    _fields_ = [("x_host", C.c_void_p), ("tsz_host", C.c_void_p), ("anchors_dev", C.c_void_p),
                ("window_dev", C.c_void_p), ("penalty_k", C.c_double), ("window_influence", C.c_double),
                ("flags", C.c_int32), ("records_host", C.c_void_p), ("refine_host", C.c_void_p),
                ("mask_col_host", C.c_void_p), ("cls_host", C.c_void_p), ("loc_host", C.c_void_p)]


class SmTrackerHp(C.Structure):
    _fields_ = [("context_amount", C.c_double), ("penalty_k", C.c_double), ("window_influence", C.c_double),
                ("lr", C.c_double), ("exemplar_size", C.c_int32), ("instance_size", C.c_int32),
                ("total_stride", C.c_int32), ("base_size", C.c_int32), ("out_size", C.c_int32), ("reserved", C.c_int32)]


# name -> (restype, argtypes); mirrors include/siammask_b200.h one to one
SIGNATURES = {
    "sm_engine_create": (C.c_int, [C.POINTER(SmConfig), C.POINTER(C.c_void_p)]),
    "sm_engine_destroy": (None, [C.c_void_p]),
    "sm_engine_load_weights": (C.c_int, [C.c_void_p, C.POINTER(SmTensorDesc), C.c_int32]),
    "sm_engine_weight_blob": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
    "sm_engine_adopt_weights": (C.c_int, [C.c_void_p]),
    "sm_engine_calibrate": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sm_engine_status": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "sm_template": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_track": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                           C.c_int32, C.c_void_p]),
    "sm_refine": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sm_track_host": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p]),
    "sm_track_host_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "sm_track_host_wait": (C.c_int, [C.c_void_p, C.c_int32]),
    "sm_crop_resize": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p]),
    "sm_warp_affine": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                 C.c_float, C.c_int32, C.c_void_p]),
    "sm_select": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [C.c_double, C.c_double] + [C.c_void_p] * 4),
    "sm_tracker_prepare": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(SmTrackerHp), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "sm_tracker_update": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(SmTrackerHp),
                                    C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sm_step": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 4 + [C.c_double, C.c_double, C.c_int32] +
                [C.c_void_p] * 9),
    "sm_template_slots": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sm_step_slots": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [C.c_double, C.c_double, C.c_int32] +
                      [C.c_void_p] * 9),
    "sm_step_slots_hp": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 6 + [C.c_int32] + [C.c_void_p] * 9),
    "sm_tracker_update_hp": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(SmTrackerHp), C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "sm_mask_iou": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 3 + [C.c_int32] * 3 +
                    [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_crop_resize_indexed": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                         C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_paste_labels": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 4 + [C.c_int32] * 3 +
                        [C.c_double, C.c_void_p, C.c_void_p]),
    "sm_paste_labels_iou": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32] * 3 +
                            [C.c_double, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_label_boxes": (C.c_int, [C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_vot_overlap": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p, C.c_void_p]),
    "sm_vot_overlap_sized": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sm_vot_trajectory_overlap": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32] +
                                  [C.c_void_p] * 6),
    "sm_vot_eao_workspace_size": (C.c_size_t, [C.c_int32, C.c_int32]),
    "sm_vot_eao_accumulate": (C.c_int, [C.c_void_p] * 3 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p] +
                              [C.c_int32] * 3 + [C.c_void_p] * 6 + [C.c_size_t, C.c_void_p]),
    "sm_crop_resize_ragged": (C.c_int, [C.c_void_p] * 4 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_warp_affine_ragged": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 3 + [C.c_int32] * 3 +
                              [C.c_float, C.c_void_p]),
    "sm_paste_labels_ragged": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32] * 3 +
                               [C.c_double, C.c_void_p, C.c_void_p]),
    "sm_paste_labels_iou_ragged": (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 6 + [C.c_int32] * 3 +
                                   [C.c_double, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "sm_label_boxes_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_void_p]),
    "sm_step_host_async": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(SmStepIO), C.c_void_p,
                                     C.POINTER(C.c_int32)]),
    "sm_xcorr_depthwise": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p]),
    "sm_conv2d": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 13 + [C.c_void_p]),
    "sm_export": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "sm_engine_set_graphs": (C.c_int, [C.c_void_p, C.c_int32]),
    "sm_profile_enable": (C.c_int, [C.c_void_p, C.c_int32]),
    "sm_profile_dump": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "sm_launch_count": (C.c_int64, [C.c_void_p]),
    "sm_engine_bytes": (C.c_size_t, [C.c_void_p]),
    "sm_last_error": (C.c_char_p, []),
    "sm_version": (C.c_char_p, []),
}

_lib = None


def load():
    """dlopen the extension (RTLD_GLOBAL not needed) and attach the prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    if not os.path.exists(LIB_PATH):
        # a fresh checkout has sources only: compile the extension in-tree (nvcc, sm_90a) — there is no other
        # implementation to fall back to, so a failed build is a hard error
        try:
            _build.build(force=True)
        except Exception as exc:
            raise ImportError(
                f"{LIB_PATH} is missing and could not be built ({exc}); build it with "
                "`python -m siammask_b200.build`. siammask_b200 has no fallback implementation.") from exc
    elif _build.is_stale():
        # sources newer than the binary: never run edited kernels against an old .so silently
        try:
            _build.build(force=True)
        except Exception as exc:
            import warnings
            warnings.warn(f"{LIB_PATH} is older than its sources and could not be rebuilt ({exc}); "
                          "running the stale binary", RuntimeWarning)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("siammask_b200: " + load().sm_last_error().decode("utf-8", "replace"))
