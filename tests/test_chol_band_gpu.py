"""The one-launch band factorisation of systems of more than 4096 unknowns (ba_chol_dataflow.cu: chol_band_kernel,
chol_backsolve_band_kernel) through bsfm_sba_Axb_Chol_factor_env, on exactly representable systems with a given row envelope
(tests/chol_band_restatement.py: A = L0 L0^T, L0 in {-1, 0, +1} inside the envelope, diagonal-block inverses I - N).  The
factor L, the 32 x 32 inverses and x must equal L0, I - N and x0 entry by entry; a mismatch names the step and the tile."""
import ctypes

import numpy as np
import pytest

from bundler_sfm_b200 import bundle
from tests import chol_band_restatement as B
from tests.chol_exact_systems import block_inverse_ref

pytestmark = pytest.mark.gpu
SUB = 32


def _lib():
    lib = bundle.load_library()
    c = ctypes
    lib.bsfm_sba_Axb_Chol_factor_env.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p,
                                                 c.c_void_p, c.POINTER(c.c_int)]
    lib.bsfm_sba_Axb_Chol_factor_env.restype = c.c_int
    lib.bsfm_ba_chol_profile.argtypes = [c.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [c.POINTER(c.c_float), c.POINTER(c.c_int), c.POINTER(c.c_double)]
    return lib


def factorise_env(A, b, first):
    """(return code, fail code, x, L, linv blocks, launches per profile class)"""
    lib = _lib()
    n = A.shape[0]
    first = np.ascontiguousarray(first, np.int32)
    x = np.full(n, np.nan)
    L = np.empty((n, n))
    linv = np.empty(((n + SUB - 1) // SUB, SUB, SUB))
    fail = ctypes.c_int(-1)
    lib.bsfm_ba_chol_profile(1)
    try:
        rc = lib.bsfm_sba_Axb_Chol_factor_env(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, first.ctypes.data, L.ctypes.data,
                                              linv.ctypes.data, None, ctypes.byref(fail))
        ms, launches, fl = (ctypes.c_float * 4)(), (ctypes.c_int * 4)(), ctypes.c_double()
        lib.bsfm_ba_chol_profile_read(ms, launches, ctypes.byref(fl))
    finally:
        lib.bsfm_ba_chol_profile(0)
    return rc, fail.value, x, L, linv, list(launches)


def workers():
    """worker CTAs of the band plan on this device: SM count - 1 (131 on an H100 SXM, 113 on an H100 PCIe)"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count - 1


def widest_fitting(n):
    w = 1
    while B.band_plan(B.tile_band_first(n, w + 1), n, workers())[0]:
        w += 1
    return w


CASES = {
    "n4097_w1": (4097, lambda: B.tile_band_first(4097, 1)),
    "n4100_jagged": (4100, lambda: B.camera_band_first(4100, 4, seed=1)),
    "n4100_w2": (4100, lambda: B.tile_band_first(4100, 2)),
    "n4100_w5": (4100, lambda: B.tile_band_first(4100, 5)),
    "n9000_jagged": (9000, lambda: B.camera_band_first(9000, 12, seed=3)),
    "n9000_widest": (9000, lambda: B.tile_band_first(9000, widest_fitting(9000))),
    "n16897_jagged": (16897, lambda: B.camera_band_first(16897, 8, seed=5)),
}


def _check_band_exact(n, first, seed):
    L0, A, x0, b = B.envelope_system(first, seed=seed)
    fits = B.band_plan(first, n, workers())[0]
    assert fits
    rc, fail, x, L, linv, launches = factorise_env(A, b, first)
    assert (rc, fail) == (1, 0), (rc, fail)
    assert launches[0] == 1 and launches[1] == 0 and launches[2] == 0 and launches[3] == 1, launches
    env = B.envelope(first, n)
    nbk = len(env) - 1
    for rb in range(nbk):      # the factor, block row by block row over the envelope (column by column inside it)
        r0, r1, c0 = rb * SUB, min(n, rb * SUB + SUB), env[rb] * SUB
        got, want = np.tril(L[r0:r1, c0:r1], r0 - c0), L0[r0:r1, c0:r1].toarray()
        bad = np.argwhere(~(got == want))
        if len(bad):
            i, j = bad[np.lexsort((bad[:, 0], bad[:, 1]))[0]]
            raise AssertionError(f"L[{r0 + i}, {c0 + j}] = {got[i, j]}, want {want[i, j]}: step {(c0 + j) // SUB}, tile ({rb}, {(c0 + j) // SUB}),"
                                 f" {len(bad)} wrong in block row {rb}")
    for k in range(nbk):
        k0, nb = k * SUB, min(SUB, n - k * SUB)
        assert np.array_equal(linv[k][:nb, :nb], block_inverse_ref(L0, k0, nb)), f"inverse of diagonal tile {k}"
    wrong = np.nonzero(x != x0)[0]
    assert len(wrong) == 0, f"x[{wrong[0]}] = {x[wrong[0]]}, want {x0[wrong[0]]} (step {wrong[0] // SUB} of the back substitution)"


@pytest.mark.parametrize("case", sorted(CASES))
def test_band_factor_is_exact(case):
    n, first = CASES[case]
    _check_band_exact(n, first(), seed=11)


def test_zero_pivot_is_failure_code_1():
    n = 4100
    first = B.tile_band_first(n, 3)
    L0, A, x0, b = B.envelope_system(first, seed=7, zero_pivots=(2500,))
    rc, fail, x, L, linv, launches = factorise_env(A, b, first)
    assert launches[0] == 1 and launches[2] == 0
    assert (rc, fail) == (0, 1)


def test_precision_bound_on_random_banded_systems():
    """|A - fl(L L^T)| <= 4 (n + 1) u |L| |L|^T on well-conditioned random systems with a jagged envelope"""
    rng = np.random.default_rng(5)
    n = 4501
    first = B.camera_band_first(n, 10, seed=6)
    keep = (np.arange(n)[None, :] >= first[:, None]) & (np.arange(n)[None, :] < np.arange(n)[:, None])
    low = np.where(keep, rng.uniform(-1.0, 1.0, (n, n)), 0.0)
    A = low + low.T
    A += np.diag(np.abs(A).sum(axis=1) + 1.0)      # diagonally dominant: SPD and well conditioned
    b = rng.standard_normal(n)
    rc, fail, x, L, linv, launches = factorise_env(A, b, first)
    assert (rc, fail) == (1, 0) and launches[0] == 1 and launches[2] == 0
    Lt = np.tril(L)
    u = np.finfo(np.float64).eps / 2
    err = np.abs(A - Lt @ Lt.T)
    bound = 4 * (n + 1) * u * (np.abs(Lt) @ np.abs(Lt).T)
    assert np.all(err <= bound + 1e-300)
    assert np.linalg.norm(A @ x - b) <= 1e-10 * np.linalg.norm(b)


@pytest.mark.parametrize("n", [1537, 4096])
def test_mid_size_banded_systems_keep_the_panel_path(n):
    """systems of at most 4096 unknowns keep the panel path whatever their envelope, with the exact answer"""
    first = B.tile_band_first(n, 2)
    assert not B.band_plan(first, n, workers())[0]
    L0, A, x0, b = B.envelope_system(first, seed=5)
    rc, fail, x, L, linv, launches = factorise_env(A, b, first)
    assert (rc, fail) == (1, 0)
    assert launches[1] > 0 and launches[2] > 0, launches
    assert np.array_equal(x, x0.astype(np.float64))


def test_wide_envelope_takes_the_panel_path():
    """a plan that does not fit (every row reaches column 0) runs the panel path on the same entry, with the same results"""
    n = 4500
    first = np.zeros(n, np.int32)
    assert not B.band_plan(first, n, workers())[0]
    L0, A, x0, b = B.envelope_system(B.tile_band_first(n, 4), seed=3)
    rc, fail, x, L, linv, launches = factorise_env(A, b, first)
    assert (rc, fail) == (1, 0)
    assert launches[1] > 0 and launches[2] > 0, launches
    assert np.array_equal(x, x0.astype(np.float64))
