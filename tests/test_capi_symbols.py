"""The C-ABI library loads on a CPU-only box and exports every symbol include/psd_b200.h
declares (no compute calls here)."""

import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "psd_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(psd_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_boundary():
    syms = declared_symbols()
    for must in ("psd_engine_create", "psd_engine_submit_host", "psd_engine_submit_device",
                 "psd_engine_set_halo_device", "psd_scan_content", "psd_scan_adaptive",
                 "psd_scan_hist_correl", "psd_last_error"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from pyscenedetect_b200 import _capi
    assert os.path.exists(_capi.LIB_PATH), "run `python __graft_entry__.py` to build the library"
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in psd_b200.h but not exported"
    assert set(_capi.SIGNATURES) == set(declared_symbols()), "ctypes table out of sync with the header"


def test_binding_loads_and_reports_errors_without_gpu():
    from pyscenedetect_b200 import _capi
    lib = _capi.load()
    assert lib.psd_abi_version() == 1
    assert b"sm_90a" in lib.psd_version()
    if lib.psd_device_count() == 0:
        # no CPU fallback: constructing an engine must fail loudly
        from pyscenedetect_b200.engine import F_HSV, Engine
        with pytest.raises(RuntimeError) as ei:
            Engine(64, 36, F_HSV)
        assert "no CUDA device" in str(ei.value) or "CUDA" in str(ei.value)


def test_config_struct_layout():
    from pyscenedetect_b200 import _capi
    assert ctypes.sizeof(_capi.PsdConfig) == 64
    assert _capi.SUMS_DTYPE.itemsize == 64


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "pyscenedetect_b200")
    for dirpath, _dirs, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "import cv2" not in src, f"{f}: product path must not call cv2"
