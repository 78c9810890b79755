"""Tile edges of the large Cholesky's persistent trailing update (ba_chol_large.cu, chol_syrk_dmma_kernel), through
bsfm_sba_Axb_Chol against LAPACK with the error bounds of test_ba_gpu.py::test_axb_chol_vs_lapack:
  1537  smallest size on the 256-column path, n = 1 (mod 256); every launch has fewer tiles than the GPU has SMs
  2560  n + 1 = 1 (mod 128): the last tile row of every panel's update holds only the right-hand-side row
  3073  odd n = 1 (mod 256): odd matrix pitch (scalar output path), last tile row again only the right-hand side"""
import ctypes

import numpy as np
import pytest

from bundler_sfm_b200 import bundle
from tests.reference_inputs import spd

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [1537, 2560, 3073])
def test_trailing_update_tile_edges_vs_lapack(n):
    A = spd(n, seed=n)
    xt = np.random.default_rng(1).standard_normal(n)
    b = A @ xt
    lib = bundle.load_library()
    fn = lib.bsfm_sba_Axb_Chol
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    fn.restype = ctypes.c_int
    x = np.zeros(n)
    assert fn(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, 0) == 1
    xr = np.linalg.solve(A, b)
    nrm = np.linalg.norm(A, 'fro')
    res = np.linalg.norm(A @ x - b) / (nrm * np.linalg.norm(x))
    res_ref = np.linalg.norm(A @ xr - b) / (nrm * np.linalg.norm(xr))
    assert res <= max(10.0 * res_ref, 1e-14), (n, res, res_ref)
    err, err_ref = np.linalg.norm(x - xt) / np.linalg.norm(xt), np.linalg.norm(xr - xt) / np.linalg.norm(xt)
    assert err <= max(20.0 * err_ref, 1e-10), (n, err, err_ref)
