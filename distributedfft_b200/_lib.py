"""ctypes binding of libdfft.so (the C ABI declared in include/dfft.h).

The product path has no fallback: if the shared library is missing this module raises at import of the
first symbol (build it with `python -m distributedfft_b200.build` or `__graft_entry__.build()`).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DFFT_LIB") or os.path.join(_HERE, "libdfft.so")  # DFFT_LIB: experimental build variants

UNIQUE_ID_BYTES = 128

SUCCESS = 0


class DfftError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"dfft error {code}: {msg}")
        self.code = code


class dfft_config(C.Structure):
    # struct Configurations, /root/reference/include/params.hpp:85-93
    _fields_ = [
        ("cuda_aware", C.c_int),
        ("warmup_rounds", C.c_int),
        ("comm_method", C.c_int),
        ("send_method", C.c_int),
        ("benchmark_dir", C.c_char_p),
        ("comm_method2", C.c_int),
        ("send_method2", C.c_int),
    ]


_lib = None

# name -> (restype, argtypes); every symbol include/dfft.h declares
SIGNATURES = {
    "dfft_get_unique_id": (C.c_int, [C.c_void_p]),
    "dfft_comm_create": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_comm_destroy": (C.c_int, [C.c_void_p]),
    "dfft_comm_rank": (C.c_int, [C.c_void_p]),
    "dfft_comm_size": (C.c_int, [C.c_void_p]),
    "dfft_plan_create": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                   C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_create_batched": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                           C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_get_batch": (C.c_size_t, [C.c_void_p]),
    "dfft_plan_create_inplace": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                           C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_is_inplace": (C.c_int, [C.c_void_p]),
    "dfft_plan_create_r2r": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.POINTER(C.c_int), C.c_size_t, C.c_size_t,
                                       C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_get_r2r_kinds": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "dfft_plan_create_padded": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                          C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t,
                                          C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_get_spectral_size": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_plan_create_pruned": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                          C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_size_t, C.c_size_t, C.c_size_t,
                                          C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_get_data_size": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_plan_create_1d": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p)]),
    "dfft_plan_create_1d_natural": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_size_t, C.POINTER(C.c_size_t),
                                              C.POINTER(C.c_void_p)]),
    "dfft_plan_get_1d_factors": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_plan_create_interleaved": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                               C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_get_components": (C.c_size_t, [C.c_void_p]),
    "dfft_plan_create_boxes": (C.c_int, [C.c_void_p, C.POINTER(dfft_config), C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t,
                                         C.c_size_t, C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_size_t,
                                         C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_set_scale": (C.c_int, [C.c_void_p, C.c_double, C.c_double]),
    "dfft_plan_get_scale": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "dfft_plan_set_weights": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "dfft_plan_get_weights": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "dfft_plan_destroy": (C.c_int, [C.c_void_p]),
    "dfft_set_work_area": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_exec_r2c": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_exec_c2r": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_exec_c2c": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "dfft_exec_r2c_partial": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "dfft_exec_c2r_partial": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "dfft_exec_c2c_partial": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "dfft_exec_r2c_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_exec_c2r_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_exec_c2c_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "dfft_exec_r2r": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "dfft_exec_r2r_partial": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "dfft_exec_r2r_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "dfft_plan_set_transform_axes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "dfft_plan_get_transform_axes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "dfft_plan_set_strides": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    "dfft_plan_get_strides": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    "dfft_plan_wait": (C.c_int, [C.c_void_p]),
    "dfft_get_in_size": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_get_in_start": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_get_out_size": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_get_out_start": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfft_get_partial_size": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_size_t)]),
    "dfft_get_partial_start": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_size_t)]),
    "dfft_get_domain_size": (C.c_size_t, [C.c_void_p]),
    "dfft_get_work_size_device": (C.c_size_t, [C.c_void_p]),
    "dfft_get_work_size_host": (C.c_size_t, [C.c_void_p]),
    "dfft_get_work_area_device": (C.c_void_p, [C.c_void_p]),
    "dfft_get_rank": (C.c_int, [C.c_void_p]),
    "dfft_get_world_size": (C.c_int, [C.c_void_p]),
    "dfft_partition": (C.c_int, [C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "dfft_layout": (C.c_int, [C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_int,
                              C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "dfft_timer_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "dfft_get_phase_count": (C.c_int, [C.c_void_p]),
    "dfft_get_phase_name": (C.c_char_p, [C.c_void_p, C.c_int]),
    "dfft_get_phase_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_int]),
    "dfft_get_last_breakdown": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "dfft_get_last_launch_count": (C.c_int, [C.c_void_p]),
    "dfft_timer_gather": (C.c_int, [C.c_void_p]),
    "dfft_get_step_count": (C.c_int, [C.c_void_p]),
    "dfft_get_step_label": (C.c_char_p, [C.c_void_p, C.c_int]),
    "dfft_get_step_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_int]),
    "dfft_timer_csv_path": (C.c_char_p, [C.c_void_p]),
    "dfft_plan_tune": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "dfft_plan_tune_report": (C.c_char_p, [C.c_void_p]),
    "dfft_get_timeline": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_int]),
    "dfft_get_timeline_label": (C.c_char_p, [C.c_void_p, C.c_int]),
    "dfft_last_error_string": (C.c_char_p, []),
    "dfft_version": (C.c_int, []),
    "dfft_fft1d_contig": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                    C.c_size_t, C.c_void_p]),
    "dfft_comm_create_dry": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "dfft_plan_describe": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfft_debug_run_step": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.POINTER(C.c_void_p), C.c_size_t, C.c_void_p,
                                      C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dfft_fft1d_general": (C.c_int, [C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.POINTER(C.c_longlong),
                                     C.c_void_p, C.POINTER(C.c_longlong), C.c_void_p]),
    "dfft_fft1d_strided": (C.c_int, [C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfft_fft1d_r2r": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
}


def lib():
    """Load libdfft.so once; raise loudly if it was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -m distributedfft_b200.build` "
                "(there is no CPU fallback).")
        l = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            f = getattr(l, name)
            f.restype = res
            f.argtypes = args
        _lib = l
    return _lib


def check(code: int) -> int:
    if code < 0:
        raise DfftError(code, (lib().dfft_last_error_string() or b"").decode())
    return code
