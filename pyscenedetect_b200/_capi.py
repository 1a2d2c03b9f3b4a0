"""ctypes binding of include/psd_b200.h (the C-ABI of libpsd_b200.so).

The library is the product: if it is missing or cannot be loaded this module raises - there is
no CPU fallback anywhere in the package.
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpsd_b200.so")

PSD_OK = 0
PSD_ERR_INVALID = -1
PSD_ERR_CUDA = -2
PSD_ERR_OOM = -3
PSD_ERR_STATE = -4
PSD_ERR_NODEVICE = -5

F_HSV = 1
F_BGRSUM = 2
F_YHIST = 4
F_EDGES = 8
F_HASH = 16
HASH_WORDS = 4
SUBMIT_PINNED = 1


def hash_words(size: int) -> int:
    """PSD_HASH_WORDS_FOR(size): uint64 words per frame of every hash array, max(4, ceil(size * size / 64))."""
    return max(HASH_WORDS, (int(size) * int(size) + 63) // 64)


class PsdConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32),
        ("device", C.c_int32),
        ("src_width", C.c_int32),
        ("src_height", C.c_int32),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("features", C.c_uint32),
        ("edge_kernel_size", C.c_int32),
        ("max_batch", C.c_int32),
        ("flags", C.c_uint32),
        ("hash_size", C.c_int32),
        ("hash_lowpass", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]


class PsdFrameLayout(C.Structure):
    """psd_frame_layout: signed byte strides of frames whose base pointer addresses channel B of pixel (0,0)."""
    _fields_ = [
        ("frame_stride", C.c_int64),
        ("row_stride", C.c_int64),
        ("pixel_stride", C.c_int64),
        ("channel_stride", C.c_int64),
    ]


SWEEP_CONTENT = 0
SWEEP_ADAPTIVE = 1
SWEEP_THRESHOLD = 2
SWEEP_HISTOGRAM = 3
SWEEP_HASH = 4
SWEEP_MAX_TOLERANCES = 8


class PsdSweepCell(C.Structure):
    """psd_sweep_cell: one grid cell of psd_sweep_cuts (64 bytes)."""
    _fields_ = [
        ("kind", C.c_int32),
        ("mode", C.c_int32),
        ("metric", C.c_void_p),
        ("metric2", C.c_void_p),
        ("threshold", C.c_double),
        ("min_content_val", C.c_double),
        ("fade_bias", C.c_double),
        ("min_frames", C.c_int64),
        ("window", C.c_int32),
        ("add_final_scene", C.c_int32),
    ]


assert C.sizeof(PsdSweepCell) == 64


# numpy view of psd_frame_sums (64 bytes)
SUMS_DTYPE = np.dtype([
    ("sad_hue", "<u8"), ("sad_sat", "<u8"), ("sad_lum", "<u8"), ("sad_edges", "<u8"),
    ("bgr_sum", "<u8"), ("has_prev", "<u8"), ("reserved", "<u8", (2,)),
])
assert SUMS_DTYPE.itemsize == 64

_vp = C.c_void_p
_i64 = C.c_int64
_i32 = C.c_int32
_u32 = C.c_uint32
_dbl = C.c_double
_dp = C.POINTER(C.c_double)

# name -> (restype, argtypes); every symbol psd_b200.h declares
SIGNATURES = {
    "psd_abi_version": (C.c_int, []),
    "psd_version": (C.c_char_p, []),
    "psd_last_error": (C.c_char_p, []),
    "psd_device_count": (C.c_int, []),
    "psd_device_info": (C.c_int, [C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_int),
                                   C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]),
    "psd_device_pci_bus_id": (C.c_int, [C.c_int, C.c_char_p, C.c_size_t]),
    "psd_launch_count": (C.c_uint64, []),
    "psd_host_alloc": (C.c_int, [C.c_size_t, C.POINTER(_vp)]),
    "psd_host_free": (C.c_int, [_vp]),
    "psd_device_alloc": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(_vp)]),
    "psd_device_free": (C.c_int, [C.c_int, _vp]),
    "psd_memcpy_h2d": (C.c_int, [C.c_int, _vp, _vp, C.c_size_t]),
    "psd_memcpy_d2h": (C.c_int, [C.c_int, _vp, _vp, C.c_size_t]),
    "psd_engine_create": (C.c_int, [C.POINTER(PsdConfig), C.POINTER(_vp)]),
    "psd_engine_destroy": (None, [_vp]),
    "psd_engine_reset": (C.c_int, [_vp]),
    "psd_engine_set_halo_host": (C.c_int, [_vp, _vp, _i64]),
    "psd_engine_set_halo_device": (C.c_int, [_vp, _vp]),
    "psd_engine_submit_host": (C.c_int, [_vp, _vp, _i64, _i64, _i64, _u32]),
    "psd_engine_submit_device": (C.c_int, [_vp, _vp, _i64, _i64]),
    "psd_engine_submit_device_layout": (C.c_int, [_vp, _vp, _i64, C.POINTER(PsdFrameLayout)]),
    "psd_engine_sync": (C.c_int, [_vp]),
    "psd_engine_compute_stream": (_vp, [_vp]),
    "psd_engine_frame_count": (_i64, [_vp]),
    "psd_engine_read_sums": (C.c_int, [_vp, _i64, _i64, _vp]),
    "psd_engine_read_yhist": (C.c_int, [_vp, _i64, _i64, _vp]),
    "psd_engine_read_hash": (C.c_int, [_vp, _i64, _i64, _vp]),
    "psd_engine_device_results": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_vp)]),
    "psd_engine_device_hash": (C.c_int, [_vp, C.POINTER(_vp)]),
    "psd_engine_timing_reset": (C.c_int, [_vp]),
    "psd_engine_timing_ms": (C.c_int, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                        C.POINTER(C.c_uint64)]),
    "psd_engine_edge_kernel_size": (C.c_int, [_vp]),
    "psd_engine_add_edge_kernel_size": (C.c_int, [_vp, _i32, C.POINTER(_i32)]),
    "psd_engine_add_hash_geometry": (C.c_int, [_vp, _i32, _i32, C.POINTER(_i32)]),
    "psd_engine_edge_kernel_size_at": (C.c_int, [_vp, _i32]),
    "psd_engine_device_edge_sads": (C.c_int, [_vp, _i32, C.POINTER(_vp)]),
    "psd_engine_device_hash_at": (C.c_int, [_vp, _i32, C.POINTER(_vp)]),
    "psd_engine_read_hash_at": (C.c_int, [_vp, _i32, _i64, _i64, _vp]),
    "psd_engine_debug_plane": (C.c_int, [_vp, C.c_int, _i64, _vp, C.c_size_t]),
    "psd_scan_content": (C.c_int, [_vp, _i64, _i64, _dp, _dbl, _vp, _vp, _vp]),
    "psd_scan_content_edges": (C.c_int, [_vp, _vp, _i64, _i64, _dp, _dbl, _vp, _vp, _vp]),
    "psd_scan_adaptive": (C.c_int, [_vp, _i64, _i32, _dbl, _vp, _vp]),
    "psd_scan_average": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "psd_scan_hist_correl": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "psd_scan_hash_dist": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "psd_scan_compare": (C.c_int, [_vp, _i64, _dbl, _i32, _vp, _vp]),
    "psd_cuts_flash_filter": (C.c_int, [_vp, _i64, _i64, _i64, _i32, _vp, _vp, _i32, _vp]),
    "psd_cuts_adaptive": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _dbl, _dbl, _i64, _vp, _vp, _i32, _vp]),
    "psd_cuts_histogram": (C.c_int, [_vp, _i64, _i64, _dbl, _i64, _vp, _vp, _i32, _vp]),
    "psd_cuts_hash": (C.c_int, [_vp, _i64, _i64, _dbl, _i64, _vp, _vp, _i32, _vp]),
    "psd_cuts_threshold": (C.c_int, [_vp, _i64, _i64, _dbl, _i32, _dbl, _i64, _i32, _vp, _vp, _i32, _vp]),
    "psd_sweep_cuts": (C.c_int, [_vp, _i32, _i64, _i64, _vp, _vp, _i32, _vp]),
    "psd_sweep_eval": (C.c_int, [_vp, _vp, _i32, _i32, _i64, _vp, _i32, _vp, _i32, _vp, _i32, _vp, C.c_size_t,
                                 _vp, _vp, _vp, _vp]),
    "psd_clip_fill": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _i32, _dbl, _vp]),
    "psd_clip_cuts": (C.c_int, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp]),
    "psd_clip_eval": (C.c_int, [_vp, _vp, _i32, _i32, _i64, _i64, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _vp,
                                C.c_size_t, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "psd_engine_scan_content_host": (C.c_int, [_vp, _i64, _i64, _dp, _dbl, _vp, _vp]),
    "psd_engine_scan_adaptive_host": (C.c_int, [_vp, _vp, _i64, _i32, _dbl, _vp]),
    "psd_engine_scan_average_host": (C.c_int, [_vp, _i64, _i64, _vp]),
    "psd_engine_scan_hist_correl_host": (C.c_int, [_vp, _i64, _i64, _i32, _vp]),
    "psd_engine_scan_hash_dist_host": (C.c_int, [_vp, _i64, _i64, _vp]),
    "psd_engine_scan_content_host_at": (C.c_int, [_vp, _i32, _i64, _i64, _dp, _dbl, _vp, _vp]),
    "psd_engine_scan_hash_dist_host_at": (C.c_int, [_vp, _i32, _i64, _i64, _vp]),
    "psd_synth_frames": (C.c_int, [C.c_int, _vp, _vp, _i64, _i32, _i32, _i64, _vp]),
    "psd_gather_bgr": (C.c_int, [C.c_int, _vp, C.POINTER(PsdFrameLayout), _i64, _i32, _i32, _vp, _i64, _vp]),
    "psd_test_hsv": (C.c_int, [C.c_int, _vp, _i64, _vp, _vp, _vp, _vp]),
    "psd_test_hash_stages": (C.c_int, [C.c_int, _vp, _i64, _i32, _i32, _i64, _vp, _i32, _vp, _vp, _vp, _vp]),
}

_lib = None


class PsdError(RuntimeError):
    """A CUDA/driver failure reported by libpsd_b200.so."""


def load():
    """Load libpsd_b200.so and bind every symbol.  Raises (never falls back) when missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python __graft_entry__.py` "
            "(pyscenedetect_b200 has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.psd_abi_version() != 1:
        raise ImportError("libpsd_b200.so ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    return load().psd_last_error().decode("utf-8", "replace")


def check(rc: int, what: str = "") -> None:
    """Map a status code to the exception types the reference detectors use:
    argument errors -> ValueError, everything else -> RuntimeError (SURVEY.md §8b)."""
    if rc == PSD_OK:
        return
    msg = last_error()
    if rc == PSD_ERR_INVALID:
        raise ValueError(f"{what}: {msg}" if what else msg)
    if rc == PSD_ERR_OOM:
        raise MemoryError(f"{what}: {msg}" if what else msg)
    raise PsdError(f"{what}: {msg}" if what else msg)
