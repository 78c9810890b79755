"""The large Cholesky's skip of all-zero panel blocks (ba_chol_large.cu: the zero flags of chol_trsm_kernel, the kept-tile
list of chol_syrk_dmma_kernel), through bsfm_sba_Axb_Chol on the block-sparse systems of tests/chol_sparse_systems.py:
  - the solution is bit-identical to the one computed before the skip existed (tests/golden/chol_sparse_golden.npz,
    written by tests/golden/make_chol_sparse_golden.py) and within the residual bound of test_chol_trailing_gpu.py
  - the profile's fp64_flops counts the tiles executed, restated here from numpy's factor (a structural zero of the
    factor is an exact zero there too); a dense system executes the whole triangle
  - a matrix that is not positive definite, or has a NaN in a nonzero block, still fails (returns 0)"""
import ctypes
import os

import numpy as np
import pytest
from scipy.linalg import solve_triangular

from bundler_sfm_b200 import bundle
from tests.chol_sparse_systems import CASES, case_system, system
from tests.reference_inputs import spd

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "chol_sparse_golden.npz")
PANEL, SLAB, TILE = 256, 64, 128
TAIL_MAX = 640      # the last panels go to the one-launch dataflow factorisation (ba_chol_large.cu, tail_fits)


def _lib():
    lib = bundle.load_library()
    lib.bsfm_sba_Axb_Chol.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    lib.bsfm_sba_Axb_Chol.restype = ctypes.c_int
    lib.bsfm_ba_chol_profile.argtypes = [ctypes.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    return lib


def _solve(A, b, profile=False):
    """(return code, x, executed trailing-update FLOPs or None)"""
    lib = _lib()
    n = A.shape[0]
    x = np.zeros(n)
    if profile:
        lib.bsfm_ba_chol_profile(1)
    try:
        rc = lib.bsfm_sba_Axb_Chol(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, 0)
        flops = None
        if profile:
            ms = (ctypes.c_float * 4)(); launches = (ctypes.c_int * 4)(); fl = ctypes.c_double()
            lib.bsfm_ba_chol_profile_read(ms, launches, ctypes.byref(fl))
            flops = fl.value
    finally:
        if profile:
            lib.bsfm_ba_chol_profile(0)
    return rc, x, flops


def _panels(n):
    """first columns k1 of the trailing updates the 256-column path runs before the dataflow tail takes over"""
    out = []
    for k0 in range(0, n, PANEL):
        if 0 < k0 and 2 * 32 < n - k0 <= TAIL_MAX:
            break
        if k0 + PANEL < n:
            out.append(k0 + PANEL)
    return out


def _executed_flops(nonzero, n):
    """nonzero: (n + 1) x n, the factor's nonzero pattern with the right-hand-side row (forward substitution) as row n.
    Per panel: a 128-row block is kept when one of its two 64-row slabs has a nonzero; the tiles are the lower triangle of
    the kept blocks; each tile counts its lower-triangle elements (right-hand-side row included) x 2 x 256."""
    nrows, elements = n + 1, 0
    for k1 in _panels(n):
        k0 = k1 - PANEL
        slab = [bool(nonzero[r:r + SLAB, k0:k1].any()) for r in range(k1, nrows, SLAB)]
        kept = [i for i in range((nrows - k1 + TILE - 1) // TILE) if any(slab[2 * i:2 * i + 2])]
        ncb = (n - k1 + TILE - 1) // TILE
        for j in (j for j in kept if j < ncb):
            c = np.arange(k1 + TILE * j, min(k1 + TILE * (j + 1), n))
            for i in (i for i in kept if i >= j):
                r0, r1 = k1 + TILE * i, min(k1 + TILE * (i + 1), nrows)
                elements += int(np.maximum(0, r1 - np.maximum(r0, c)).sum())
    return 2.0 * PANEL * elements


def _dense_flops(n):
    return sum(2.0 * PANEL * ((n - k1) * (n - k1 + 1) // 2 + (n - k1)) for k1 in _panels(n))


def _residual_ok(A, b, x):
    xr = np.linalg.solve(A, b)
    nrm = np.linalg.norm(A, 'fro')
    res = np.linalg.norm(A @ x - b) / (nrm * np.linalg.norm(x))
    res_ref = np.linalg.norm(A @ xr - b) / (nrm * np.linalg.norm(xr))
    return res <= max(10.0 * res_ref, 1e-14), (res, res_ref)


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_sparse_solution_bits_and_flops(name):
    A, b = case_system(name)
    n = A.shape[0]
    rc, x, flops = _solve(A, b, profile=True)
    assert rc == 1
    want = np.load(GOLDEN)[name]
    assert x.tobytes() == want.tobytes(), (name, int(np.count_nonzero(x != want)), float(np.abs(x - want).max()))
    ok, info = _residual_ok(A, b, x)
    assert ok, (name, info)
    L = np.linalg.cholesky(A)
    y = solve_triangular(L, b, lower=True)
    nonzero = np.vstack([L, y[None, :]]) != 0
    assert flops == _executed_flops(nonzero, n), (name, flops, _executed_flops(nonzero, n), _dense_flops(n))


def test_dense_system_executes_whole_triangle():
    n = 2560
    A = spd(n, seed=5)
    b = np.random.default_rng(2).standard_normal(n)
    rc, x, flops = _solve(A, b, profile=True)
    assert rc == 1
    assert flops == _dense_flops(n) == _executed_flops(np.ones((n + 1, n), bool), n)


def test_sparse_not_positive_definite_fails():
    A, b = system("band", 2560, seed=11)
    A[2000, 2000] = -A[2000, 2000]
    assert _solve(A, b)[0] == 0


def test_sparse_nan_in_nonzero_block_fails():
    A, b = system("band", 2560, seed=12)
    r, c = 9 * 101 + 3, 9 * 100 + 2          # cameras 100 and 101 share points: a nonzero block
    assert A[r, c] != 0
    A[r, c] = A[c, r] = np.nan
    assert _solve(A, b)[0] == 0
