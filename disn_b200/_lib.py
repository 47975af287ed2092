"""ctypes binding of libdisn_b200.so (the C ABI declared in include/disn_b200.h).

There is no CPU or eager fallback: if the shared library is missing it is built with nvcc, and if that
fails -- or no sm_90 GPU is present when a context is created -- the error is raised to the caller.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdisn_b200.so")

DISN_DEVICE_PTR = 1
DISN_OBJ_PARTS = 1
DISN_ERR_OBJ_UNSUPPORTED = -5
PREC_FP32 = 0
PREC_BF16X3 = 1
PREC_F16F8 = 2


class DisnConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32), ("vgg_in", C.c_int32),
                ("num_classes", C.c_int32), ("clamp_max", C.c_float), ("sdf_weight", C.c_float),
                ("tanh_out", C.c_int32), ("precision", C.c_int32), ("max_batch", C.c_int32)]


EXPORTS = {
    # name: (restype, argtypes)
    "disn_default_config": (None, [C.POINTER(DisnConfig)]),
    "disn_create": (C.c_int, [C.POINTER(DisnConfig), C.POINTER(C.c_void_p)]),
    "disn_destroy": (None, [C.c_void_p]),
    "disn_last_error": (C.c_char_p, []),
    "disn_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "disn_synchronize": (C.c_int, [C.c_void_p]),
    "disn_set_precision": (C.c_int, [C.c_void_p, C.c_int32]),
    "disn_load_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32]),
    "disn_finalize_weights": (C.c_int, [C.c_void_p]),
    "disn_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_uint32]),
    "disn_get_encoded": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
    "disn_eval_points": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64,
                                   C.c_void_p, C.c_void_p, C.c_uint32]),
    "disn_eval_grid": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_void_p, C.c_uint32]),
    "disn_write_dist": (C.c_int, [C.c_char_p, C.c_int32, C.POINTER(C.c_double), C.c_void_p]),
    "disn_cam_estimate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "disn_cam_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_nn_distance": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_write_obj": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]),
    "disn_marching_cubes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_float,
                                      C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int64),
                                      C.c_uint32]),
    "disn_launch_count": (C.c_int64, [C.c_void_p]),
    "disn_eval_grid_resident": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_int32, C.c_int32,
                                          C.POINTER(C.c_void_p)]),
    "disn_eval_grid_indexed": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                         C.c_int64, C.c_void_p, C.c_uint32]),
    "disn_eval_grid_adaptive": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                                          C.c_double, C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(C.c_int32)]),
    "disn_mesh_grid_adaptive": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                                          C.c_double, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                          C.POINTER(C.c_int64)]),
    "disn_mc_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_float, C.c_uint32,
                              C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "disn_mc_fetch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_mesh_counts": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "disn_mc_write_obj": (C.c_int, [C.c_void_p, C.c_char_p]),
    "disn_mesh_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]),
    "disn_mesh_clean": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.POINTER(C.c_int64),
                                  C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "disn_mesh_sdf": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_double, C.c_double, C.c_void_p,
                                C.POINTER(C.c_double), C.c_uint32]),
    "disn_mesh_sdf_phase_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "disn_mesh_part_areas": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]),
    "disn_mesh_normalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.POINTER(C.c_double), C.c_void_p]),
    "disn_field": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "disn_sdf_band_count": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_uint32, C.c_void_p]),
    "disn_sdf_band_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_sdf_strided": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_uint32, C.c_void_p]),
    "disn_fetch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "disn_shared_alloc": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_void_p), C.c_char_p]),
    "disn_shared_open": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "disn_shared_close": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "disn_approx_match": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "disn_match_cost": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "disn_iou": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                           C.c_int64, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p, C.c_void_p]),
    "disn_iou_views": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_eval_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_uint32]),
    "disn_eval_points_ex": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_point_img_feat": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "disn_obj_read": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                C.POINTER(C.c_int32)]),
    "disn_obj_parts": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]),
    "disn_obj_read_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "disn_sdf_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_float,
                                   C.c_float, C.c_float, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

# diagnostics (include/disn_b200_test.h), exported by libdisn_b200_test.so only
TEST_EXPORTS = {
    "disn_debug_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "disn_tc_stream_probe": (C.c_int, [C.c_int]),
    "disn_tc_op_probe": (C.c_int, [C.c_int]),
    "disn_tc_selftest": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "disn_tc_selftest_mixed": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "disn_debug_tc_weights": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "disn_adaptive_mask": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "disn_adaptive_from_field": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_float, C.c_double,
                                           C.c_uint32, C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(C.c_int32)]),
    "disn_adaptive_phase_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "disn_mesh_adaptive_from_field": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_float,
                                                C.c_double, C.c_uint32, C.c_void_p, C.POINTER(C.c_int32),
                                                C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "disn_mesh_adaptive_phase_ms": (C.c_int, [C.c_void_p, C.c_void_p]),
    "disn_mesh_adaptive_bytes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "disn_mesh_adaptive_edges": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "disn_debug_obj_tokens": (C.c_int, [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "disn_debug_cam_heads": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None
_test_lib = None
TEST_LIB_PATH = os.path.join(HERE, "libdisn_b200_test.so")



def load(build_if_missing: bool = True):
    """Load (building first if needed) the native library; raises if it cannot be produced."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _build
        if _build.needs_build():
            _build.build()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libdisn_b200.so is missing (%s): build it with `python -m disn_b200.build`; "
                           "there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)     # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def load_test():
    """The diagnostics library (selftests, probes, debug GEMM harness) -- tests/ and tools/ only."""
    global _test_lib
    if _test_lib is not None:
        return _test_lib
    load()
    if not os.path.exists(TEST_LIB_PATH):
        raise RuntimeError("libdisn_b200_test.so is missing: build it with `python -m disn_b200.build`")
    lib = C.CDLL(TEST_LIB_PATH)
    for table in (EXPORTS, TEST_EXPORTS):
        for name, (res, args) in table.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
    _test_lib = lib
    return lib


class DisnError(RuntimeError):
    pass


def check(rc: int):
    if rc != 0:
        raise DisnError("%s (rc=%d)" % (load().disn_last_error().decode("utf-8", "replace"), rc))
