"""CPU tests (no GPU): the C-ABI library loads, exports every symbol include/*.h declares, and its
compute entry points fail loudly (no CPU fallback) when no CUDA device is present."""
import ctypes
import glob
import os
import re

import numpy as np
import pytest

import bundler_sfm_b200
from bundler_sfm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# include/bsfm_b200_sba.h declares what the link-time replacements of libsba / libsfmdrv export (shim/_build), the other
# headers what libbsfm_b200.so exports
SHIM_HEADERS = {"bsfm_b200_sba.h"}


def declared_symbols(shim=False):
    names = []
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        if (os.path.basename(h) in SHIM_HEADERS) != shim:
            continue
        src = open(h).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        src = re.sub(r"//[^\n]*", "", src)
        for m in re.finditer(r"\b((?:bsfm|sba|sfm|run)_[A-Za-z0-9_]*)\s*\(", src):
            names.append(m.group(1))
    return sorted(set(names))


def test_library_loads_and_exports_all_declared_symbols():
    lib = bundler_sfm_b200.load_library()
    syms = declared_symbols()
    assert "bsfm_match_pair" in syms and "bsfm_match_run" in syms
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing
    assert b"sm_90a" in lib.bsfm_version()


def test_shim_libraries_export_the_reference_driver_symbols():
    """libsba_b200.so / libsfmdrv_b200.so: the reference's sba drivers, run_sfm and the sfm-driver projection callbacks"""
    build = os.path.join(ROOT, "shim", "_build")
    if not os.path.exists(os.path.join(build, "libsba_b200.so")):
        pytest.skip("shim/_build not built")
    bundler_sfm_b200.load_library()     # the shims link against libbsfm_b200.so (rpath)
    drv = ctypes.CDLL(os.path.join(build, "libsfmdrv_b200.so"), mode=ctypes.RTLD_GLOBAL)
    sba = ctypes.CDLL(os.path.join(build, "libsba_b200.so"))
    for name in ("sba_motstr_levmar_x", "sba_motstr_levmar", "sba_mot_levmar_x", "sba_mot_levmar"):
        assert hasattr(sba, name), name
    for name in ("run_sfm", "sfm_project_point3", "sfm_project_point3_mot"):
        assert hasattr(drv, name), name
    for name in declared_symbols(shim=True):
        assert hasattr(sba, name) or hasattr(drv, name), name


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_compute_fails_loudly_without_gpu():
    lib = bundler_sfm_b200.load_library()
    k = np.zeros((4, 128), np.uint8)
    out = np.zeros((4, 2), np.int32)
    rc = lib.bsfm_match_pair(k.ctypes.data, 4, k.ctypes.data, 4, 0.6, out.ctypes.data, 4)
    assert rc < 0
    assert b"no CPU fallback" in lib.bsfm_last_error() or b"CUDA" in lib.bsfm_last_error()
    off = np.array([0, 4], np.int64)
    h = lib.bsfm_keydb_create(k.ctypes.data, off.ctypes.data, 1)
    assert not h
    A, L = np.eye(4), np.zeros((4, 4))
    b, x, linv = np.ones(4), np.zeros(4), np.zeros((1, 32, 32))
    fail = ctypes.c_int(-7)
    rc = lib.bsfm_sba_Axb_Chol_factor(ctypes.c_void_p(A.ctypes.data), ctypes.c_void_p(b.ctypes.data), ctypes.c_void_p(x.ctypes.data), 4,
                                      ctypes.c_void_p(L.ctypes.data), ctypes.c_void_p(linv.ctypes.data), None, ctypes.byref(fail))
    assert rc < 0 and fail.value == -7 and not x.any()


def test_pair_count_helper():
    lib = bundler_sfm_b200.load_library()
    assert lib.bsfm_match_num_pairs(500, -1) == 124750
    assert lib.bsfm_match_num_pairs(5, 2) == 0 + 1 + 2 + 2 + 2
    from bundler_sfm_b200 import keymatch
    assert len(keymatch.pair_list(5, 2)) == 7
    assert keymatch.pair_list(3) == [(0, 1), (0, 2), (1, 2)]
