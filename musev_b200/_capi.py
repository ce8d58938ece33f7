"""ctypes binding of include/musev_b200.h. There is no fallback: if the library is missing, loading raises."""
from __future__ import annotations

import ctypes as C
import os

from .build import LIB_PATH

_lib = None


class MvbError(RuntimeError):
    pass


class ConvGemmDesc(C.Structure):
    _fields_ = [
        ("a0", C.c_void_p), ("c0", C.c_int),
        ("a0_stride_w", C.c_longlong), ("a0_stride_h", C.c_longlong), ("a0_stride_n", C.c_longlong),
        ("a1", C.c_void_p), ("c1", C.c_int),
        ("a1_stride_w", C.c_longlong), ("a1_stride_h", C.c_longlong), ("a1_stride_n", C.c_longlong),
        ("W", C.c_int), ("H", C.c_int), ("NF", C.c_int),
        ("ntaps", C.c_int), ("dy", C.c_int8 * 9), ("dx", C.c_int8 * 9),
        ("weight", C.c_void_p), ("N", C.c_int),
        ("out", C.c_void_p), ("ldc", C.c_longlong),
        ("bias", C.c_void_p),
        ("rowadd", C.c_void_p), ("rows_per_group", C.c_int), ("ld_rowadd", C.c_int),
        ("residual", C.c_void_p), ("ld_res", C.c_longlong),
        ("alpha", C.c_float), ("beta", C.c_float),
        ("geglu", C.c_int), ("act", C.c_int), ("out_f32", C.c_int), ("stride2", C.c_int),
    ]


class AttentionDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_longlong),
        ("NF", C.c_int), ("Nq", C.c_int), ("heads", C.c_int), ("d", C.c_int), ("dp", C.c_int),
        ("scale", C.c_float), ("nseg", C.c_int),
        ("k", C.c_void_p * 2), ("v", C.c_void_p * 2), ("ldkv", C.c_longlong * 2), ("kv_rows", C.c_longlong * 2),
        ("nk", C.c_int * 2), ("fdiv", C.c_int * 2), ("fmul", C.c_longlong * 2), ("fadd", C.c_longlong * 2),
        ("out", C.c_void_p), ("ldo", C.c_longlong),
        ("out_scale", C.c_float), ("accumulate", C.c_int), ("v_ones_col", C.c_int), ("variant", C.c_int),
    ]


def lib() -> C.CDLL:
    """Load libmusevb200.so (built in-tree by musev_b200.build). Raises if it is not there."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MvbError(
                f"{LIB_PATH} not found: build it with `python -m musev_b200.build` "
                "(musev_b200 has no CPU or PyTorch fallback)")
        _lib = C.CDLL(LIB_PATH)
        _lib.mvb_last_error.restype = C.c_char_p
        _declare(_lib)
    return _lib


def _declare(l: C.CDLL) -> None:
    l.mvb_version.restype = C.c_int
    l.mvb_op_conv_gemm.argtypes = [C.POINTER(ConvGemmDesc), C.c_void_p]
    l.mvb_op_conv_gemm.restype = C.c_int
    l.mvb_op_small_conv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    l.mvb_op_small_conv.restype = C.c_int
    l.mvb_op_attention.argtypes = [C.POINTER(AttentionDesc), C.c_void_p]
    l.mvb_op_attention.restype = C.c_int
    l.mvb_debug_attention_trace.argtypes = [C.c_void_p]
    l.mvb_debug_attention_trace.restype = C.c_int
    l.mvb_tensor_map_cache_stats.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    l.mvb_tensor_map_cache_stats.restype = C.c_int
    l.mvb_op_temporal_attention.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_float, C.c_void_p, C.c_int, C.c_void_p]
    l.mvb_op_temporal_attention.restype = C.c_int
    l.mvb_op_groupnorm.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_op_groupnorm.restype = C.c_int
    l.mvb_op_groupnorm_fused.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.POINTER(C.c_uint), C.c_void_p]
    l.mvb_op_groupnorm_fused.restype = C.c_int
    l.mvb_op_layernorm.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]
    l.mvb_op_layernorm.restype = C.c_int
    l.mvb_fuse_cfg_ddim.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_int,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_fuse_cfg_ddim.restype = C.c_int
    l.mvb_fuse_cfg_affine.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_float,
                                      C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mvb_fuse_cfg_affine.restype = C.c_int
    l.mvb_accumulate_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                        C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    l.mvb_accumulate_window.restype = C.c_int
    l.mvb_launch_count.argtypes = [C.c_int]
    l.mvb_launch_count.restype = C.c_longlong
    l.mvb_profile_enable.argtypes = [C.c_int]
    l.mvb_profile_enable.restype = None
    l.mvb_profile_collect.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
    l.mvb_profile_collect.restype = C.c_int


def check(rc: int) -> None:
    if rc != 0:
        raise MvbError(f"musev_b200 error {rc}: {lib().mvb_last_error().decode()}")


CATEGORIES = ("gemm", "attention", "temporal_attention", "groupnorm", "layernorm", "other")


def launch_count(category: int = -1) -> int:
    return int(lib().mvb_launch_count(category))


def profile_enable(on: bool) -> None:
    lib().mvb_profile_enable(int(on))


def tensor_map_cache_stats():
    """(hits, misses) of the process-wide memo of encoded TMA descriptors."""
    h, m = C.c_ulonglong(0), C.c_ulonglong(0)
    check(lib().mvb_tensor_map_cache_stats(C.byref(h), C.byref(m)))
    return int(h.value), int(m.value)


def profile_collect():
    ms = (C.c_double * 6)()
    n = (C.c_longlong * 6)()
    check(lib().mvb_profile_collect(ms, n))
    return {c: dict(ms=ms[i], launches=int(n[i])) for i, c in enumerate(CATEGORIES)}
