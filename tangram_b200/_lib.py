"""ctypes binding of include/tangram_b200.h.  There is NO CPU fallback: if the library is
missing or no sm_90 GPU is visible the calls raise."""
import ctypes
import os

import numpy as np

from . import _build

HIST_COLS = 16
PREC = {"fp32": 0, "bf16": 1, "bf16x3": 2}
DENSITY_NONE, DENSITY_CELLS, DENSITY_SOURCE = 0, 1, 2
GRAPH_VOXEL_WEIGHTS, GRAPH_NEIGHBORHOOD_FILTER, GRAPH_SPATIAL_WEIGHTS = 0, 1, 2


class Config(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_int32), ("device", ctypes.c_int32),
        ("n_cells", ctypes.c_int32), ("n_voxels", ctypes.c_int32),
        ("n_genes", ctypes.c_int32), ("n_types", ctypes.c_int32),
        ("n_cells_global", ctypes.c_int64),
        ("precision", ctypes.c_int32), ("density_mode", ctypes.c_int32),
        ("lambda_g1", ctypes.c_float), ("lambda_d", ctypes.c_float), ("lambda_g2", ctypes.c_float),
        ("lambda_r", ctypes.c_float), ("lambda_l1", ctypes.c_float), ("lambda_l2", ctypes.c_float),
        ("lambda_neighborhood_g1", ctypes.c_float), ("lambda_ct_islands", ctypes.c_float),
        ("lambda_getis_ord", ctypes.c_float),
        ("adam_beta1", ctypes.c_float), ("adam_beta2", ctypes.c_float), ("adam_eps", ctypes.c_float),
        ("constrained", ctypes.c_int32), ("lambda_count", ctypes.c_float), ("lambda_f_reg", ctypes.c_float),
        ("target_count", ctypes.c_float),
    ]


class TangramB200Error(RuntimeError):
    pass


_P = ctypes.c_void_p
_F = ctypes.POINTER(ctypes.c_float)
_I32 = ctypes.POINTER(ctypes.c_int32)
_I64 = ctypes.POINTER(ctypes.c_int64)

# name -> (restype, argtypes); mirrors include/tangram_b200.h one to one
SIGNATURES = {
    "tgb200_create": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.POINTER(_P)]),
    "tgb200_destroy": (ctypes.c_int, [_P]),
    "tgb200_set_expression": (ctypes.c_int, [_P, _P, _P, _P]),
    "tgb200_set_density": (ctypes.c_int, [_P, _P, _P, _P]),
    "tgb200_set_ct_encode": (ctypes.c_int, [_P, _P, _P]),
    "tgb200_set_graph": (ctypes.c_int, [_P, ctypes.c_int, _P, _P, _P, ctypes.c_int64, _P]),
    "tgb200_set_mapping": (ctypes.c_int, [_P, _P, _P]),
    "tgb200_init_mapping_normal": (ctypes.c_int, [_P, ctypes.c_uint64, _P]),
    "tgb200_init_mapping_normal_rows": (ctypes.c_int, [_P, ctypes.c_uint64, ctypes.c_int64, _P]),
    "tgb200_reset_adam": (ctypes.c_int, [_P, _P]),
    "tgb200_set_filter": (ctypes.c_int, [_P, _P, _P]),
    "tgb200_get_filter": (ctypes.c_int, [_P, _P, _P, _P]),
    "tgb200_run": (ctypes.c_int, [_P, ctypes.c_int32, ctypes.c_float, _P]),
    "tgb200_step_begin": (ctypes.c_int, [_P, _P]),
    "tgb200_exchange_buffer": (ctypes.c_int, [_P, ctypes.POINTER(_P), _I64]),
    "tgb200_step_end": (ctypes.c_int, [_P, ctypes.c_float, _P]),
    "tgb200_comm_unique_id": (ctypes.c_int, [_P, ctypes.c_int64]),
    "tgb200_comm_init_rank": (ctypes.c_int, [_P, _P, ctypes.c_int32, ctypes.c_int32]),
    "tgb200_set_comm": (ctypes.c_int, [_P, _P, ctypes.c_int32, ctypes.c_int32]),
    "tgb200_comm_create": (ctypes.c_int, [_P, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(_P)]),
    "tgb200_comm_destroy": (ctypes.c_int, [_P]),
    "tgb200_history_len": (ctypes.c_int, [_P, _I64]),
    "tgb200_get_history": (ctypes.c_int, [_P, ctypes.c_int64, ctypes.c_int64, _P, _P]),
    "tgb200_get_mapping": (ctypes.c_int, [_P, _P, _P]),
    "tgb200_validation_terms": (ctypes.c_int, [_P, _P, _P]),
    "tgb200_project": (ctypes.c_int, [_P, _P, ctypes.c_int64, _P, _P]),
    "tgb200_get_state": (ctypes.c_int, [_P, _P, _P, _P, _I64, _P]),
    "tgb200_set_state": (ctypes.c_int, [_P, _P, _P, _P, ctypes.c_int64, _P]),
    "tgb200_kernel_launches": (ctypes.c_int, [_P, _I64]),
    "tgb200_profile_step": (ctypes.c_int, [_P, ctypes.c_float, _P, ctypes.POINTER(ctypes.c_char_p), _F,
                                           ctypes.c_int32, _I32]),
    "tgb200_algorithmic_cost": (ctypes.c_int, [_P, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    "tgb200_debug_timeline": (ctypes.c_int, [_P, ctypes.c_int32, ctypes.POINTER(ctypes.c_char_p), _I32, _F, ctypes.c_int32, _I32]),
    "tgb200_debug_buffer": (ctypes.c_int, [_P, ctypes.c_char_p, _P, ctypes.c_int64, _I64]),
    "tgb200_host_pin": (ctypes.c_int, [_P, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32]),
    "tgb200_host_unpin": (ctypes.c_int, [_P]),
    "tgb200_last_error": (ctypes.c_char_p, []),
    "tgb200_version": (ctypes.c_char_p, []),
}

_lib = None


def load(build_if_missing=True):
    """dlopen tangram_b200/libtangram_b200.so (building it with nvcc first if needed)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if not os.path.exists(path) or (build_if_missing and _build.find_nvcc() and not _build.is_current()):
        if not build_if_missing:
            raise TangramB200Error(f"{path} is missing: run __graft_entry__.build()")
        _build.build()
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the header and the .so disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status):
    if status != 0:
        msg = load().tgb200_last_error()
        raise TangramB200Error(f"tangram_b200 error {status}: {msg.decode() if msg else '?'}")


def ptr(a):
    """Raw pointer of a numpy array (host) / torch tensor (host or device) / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(_P)
    if hasattr(a, "data_ptr"):
        return _P(a.data_ptr())
    raise TypeError(f"cannot take a pointer of {type(a)}")
