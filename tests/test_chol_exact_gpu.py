"""Every dense Cholesky path of bsfm_sba_Axb_Chol, entry by entry, on exactly representable systems
(tests/chol_exact_systems.py: A = L0 L0^T with an integer L0 whose diagonal-block inverses are I - N).  Through
bsfm_sba_Axb_Chol_factor the tests see the factor L, the 32 x 32 diagonal-block inverses (linv), the 256 x 256 panel
inverses L_pp^-T of the large path (xinv), the solution x and the raw failure word, and require each to be EXACTLY the
reference: a stale read, a race, a misplaced or wrongly skipped tile, or a wrong index shows up as a nonzero difference at
a known entry, which the assertion names (path, panel, 128-row tile, 64-row slab).  +0 and -0 count as equal.

Exact integer data would hide a reduced-precision step (fp32 and TF32 are exact on small integers), so
test_factor_precision_bound checks the factor of well-conditioned random systems against an fp64 backward-error bound."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from bundler_sfm_b200 import bundle
from tests.chol_exact_systems import (LARGE_MIN, PANEL, SLAB, SUB, TAIL_MAX, TILE, block_inverse_ref, executed_flops,
                                      exact_system, scaled, slab_flags)
from tests.reference_inputs import spd

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALES = (-40, 37)


def _lib():
    lib = bundle.load_library()
    c = ctypes
    lib.bsfm_sba_Axb_Chol_factor.argtypes = [c.c_void_p, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_void_p, c.c_void_p,
                                             c.POINTER(c.c_int)]
    lib.bsfm_sba_Axb_Chol_factor.restype = c.c_int
    lib.bsfm_ba_chol_profile.argtypes = [c.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [c.POINTER(c.c_float), c.POINTER(c.c_int), c.POINTER(c.c_double)]
    return lib


def factorise(A, b, profile=False):
    """(return code, fail code, x, L, linv blocks, xinv blocks or None, executed trailing-update FLOPs or None)"""
    lib = _lib()
    n = A.shape[0]
    x = np.full(n, np.nan)
    L = np.empty((n, n))
    linv = np.empty(((n + SUB - 1) // SUB, SUB, SUB))
    xinv = np.empty(((n + PANEL - 1) // PANEL, PANEL, PANEL)) if n > LARGE_MIN else None
    fail = ctypes.c_int(-1)
    if profile:
        lib.bsfm_ba_chol_profile(1)
    try:
        rc = lib.bsfm_sba_Axb_Chol_factor(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, L.ctypes.data, linv.ctypes.data,
                                          None if xinv is None else xinv.ctypes.data, ctypes.byref(fail))
        flops = None
        if profile:
            ms = (ctypes.c_float * 4)(); launches = (ctypes.c_int * 4)(); fl = ctypes.c_double()
            lib.bsfm_ba_chol_profile_read(ms, launches, ctypes.byref(fl))
            flops = fl.value
    finally:
        if profile:
            lib.bsfm_ba_chol_profile(0)
    return rc, fail.value, x, L, linv, xinv, flops


def path_of(n, tail_max=TAIL_MAX, dataflow=True):
    if n <= SUB:
        return "single tile (chol_step_kernel)"
    if n <= 640 and dataflow:
        return "dataflow"
    if n <= 1536:
        return "fused step" + (" + tile kernel" if n > 1248 else "")
    return f"large path (tail <= {tail_max}{'' if dataflow else ', dataflow off'})"


def _where(i, j, n):
    """the blocks that computed factor entry (i, j), i >= j"""
    p = j // PANEL
    s = f"panel {p} (columns {p * PANEL}..{min(n, p * PANEL + PANEL) - 1}), 32-tile ({i // SUB}, {j // SUB})"
    if n > LARGE_MIN:
        s += f", 128-row tile ({i // TILE}, {j // TILE}) of the trailing updates, 64-row slab {i // SLAB} of the panel solves"
    return s


def _first_wrong(got, want, lower=True):
    """(i, j) of the first mismatch, column by column (the earliest panel it shows in); None when equal as values"""
    wrong = ~(got == want)
    if lower:
        wrong = np.tril(wrong)
    if not wrong.any():
        return None, 0
    idx = np.argwhere(wrong)
    k = np.lexsort((idx[:, 0], idx[:, 1]))[0]
    return tuple(int(v) for v in idx[k]), int(wrong.sum())


_SYS = {}


def system(n, pattern="dense", seed=None, zero_pivots=()):
    """exact_system, the last one kept (the scaled variants of a case reuse its A)"""
    key = (n, pattern, seed, tuple(zero_pivots))
    if key not in _SYS:
        _SYS.clear()
        _SYS[key] = exact_system(n, pattern, seed=n if seed is None else seed, zero_pivots=zero_pivots)
    return _SYS[key]


def check_exact(n, pattern="dense", s=0, profile=False, lookahead=True, tail_max=TAIL_MAX, dataflow=True):
    """factor, inverses and solution of the exact system equal the references; with `profile` the executed FLOPs equal the
    restatement of the launches chol_solve_large makes (look-ahead, tail and dataflow settings as given)"""
    L0, A, x0, b = system(n, pattern)
    A, b = scaled(A, b, s)
    rc, fail, x, L, linv, xinv, flops = factorise(A, b, profile)
    what = f"{path_of(n, tail_max, dataflow)}, {pattern} n={n}, scale 2^{s}"
    # L: whole rows at a time (the largest case is 2 GB per matrix)
    for r0 in range(0, n, 1024):
        r1 = min(n, r0 + 1024)
        got, want = L[r0:r1], np.ldexp(L0[r0:r1].toarray().astype(np.float64), s)
        ij, cnt = _first_wrong(got, want, lower=False)      # a NaN is a wrong entry
        if ij is not None:
            i, j = ij[0] + r0, ij[1]
            part = "above the diagonal" if j > i else _where(i, j, n)
            pytest.fail(f"{what}: L[{i}, {j}] = {L[i, j]!r}, exact {want[ij]!r} ({part}); {cnt} wrong entries in rows {r0}..{r1 - 1}")
    assert fail == 0 and rc == 1, (what, "rc", rc, "fail_code", fail)
    for k in range(linv.shape[0]):
        w = min(SUB, n - SUB * k)
        want = np.ldexp(block_inverse_ref(L0, SUB * k, w).astype(np.float64), -s)
        ij, cnt = _first_wrong(linv[k, :w, :w], want, lower=False)
        if ij is not None:
            pytest.fail(f"{what}: linv block {k} (32-tile {k}, panel {SUB * k // PANEL})[{ij[0]}, {ij[1]}] = {linv[k][ij]!r}, "
                        f"exact {want[ij]!r}; {cnt} wrong")
    if xinv is not None:
        for p in range(xinv.shape[0]):
            w = min(PANEL, n - PANEL * p)
            want = np.ldexp(block_inverse_ref(L0, PANEL * p, w).T.astype(np.float64), -s)
            ij, cnt = _first_wrong(xinv[p, :w, :w], want, lower=False)
            if ij is not None:
                pytest.fail(f"{what}: xinv of panel {p} [{ij[0]}, {ij[1]}] = {xinv[p][ij]!r}, exact {want[ij]!r}; "
                            f"{cnt} wrong (64-row slab {ij[0] // SLAB} of the identity solve)")
    bad = np.nonzero(~(x == x0))[0]
    assert bad.size == 0, (what, "x", int(bad.size), "wrong, first", int(bad[0]), x[bad[0]], int(x0[bad[0]]))
    if profile:
        y = L0.T @ x0
        want = executed_flops(n, slab_flags(L0, y), lookahead, tail_max, dataflow)
        assert flops == want, (what, "fp64_flops", flops, "restated", want)


# (n, the path and edge it reaches)
SIZES = [
    (1, "single tile"), (9, "single tile"), (32, "single tile"),
    (33, "dataflow, partial tile"), (64, "dataflow"), (65, "dataflow, 1-row tile"), (97, "dataflow"),
    (450, "dataflow, two tiles per CTA"), (640, "dataflow, largest"),
    (641, "fused step, one wave"), (1024, "fused step, one wave"), (1025, "fused step, several waves"),
    (1248, "fused step, several waves"), (1249, "tile-kernel steps, 1-row last block"), (1536, "tile-kernel steps"),
    (1537, "large path, smallest"), (1547, "large path, odd pitch"),
    (2688, "tail hand-over at remainder 640"), (2689, "tail hand-over at remainder 385"),
    (2560, "right-hand-side-only last tile row"), (3073, "right-hand-side-only last tile row"),
    (4100, "dense, DESIGN.md 8 item 1"), (4500, "dense, DESIGN.md 8 item 1"), (9000, "dense, config 3"),
]


@pytest.mark.parametrize("s", [0, "scaled"])
@pytest.mark.parametrize("n", [c[0] for c in SIZES])
def test_exact_factor(n, s):
    """every entry of L, linv, xinv and x of the dense exact system, unit diagonal and scaled by 2^-40 or 2^37.
    The scaled cases of the fused-step path (n <= 32, 641..1536) are exact too: the scalar pivot chain of chol_step_kernel
    takes CUDA's rsqrt(), which is not proven exact on powers of four the way the tensor-core potf2's reciprocal square root
    is (tests/test_chol_exact_systems.py), but returned exactly 2^-s on 4^s for both scales on an H100.  A failure of only
    those cases would mean rsqrt() rounds a power of four, not a wrong factor."""
    check_exact(n, "dense", s=(0 if s == 0 else SCALES[n % 2]))


SPARSE = [("ring", 4500), ("band9", 4005), ("arrow", 3600), ("blockdiag", 2560), ("ring", 1537), ("band9", 2560),
          ("arrow", 3073), ("blockdiag", 3073)]


@pytest.mark.parametrize("s", [0, "scaled"])
@pytest.mark.parametrize("pattern,n", SPARSE)
def test_exact_factor_sparse_and_executed_flops(pattern, n, s):
    """block-sparse factors (the zero-block skip of the trailing update and the panel solve) and the FLOPs it executed"""
    check_exact(n, pattern, s=(0 if s == 0 else SCALES[n % 2]), profile=True)


@pytest.mark.parametrize("s", [0, 37])
def test_exact_factor_more_than_128_row_blocks(s):
    """n = 16897, banded L0: both launches of panel 0 and the column launch of panel 1 have more than 128 row blocks and
    keep every tile; all later launches use the kept-tile list.  FLOPs restated with the look-ahead split"""
    check_exact(16897, "band", s=s, profile=True)


def _child(env, calls):
    """run check_exact(**kw) for every kw in `calls` in a child process with `env` (the switches are read once per process)"""
    code = ("import sys; sys.path.insert(0, %r); from tests.test_chol_exact_gpu import check_exact\n"
            "for kw in %r: check_exact(**kw)") % (ROOT, calls)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **env))
    assert r.returncode == 0, (env, r.stderr[-3000:])


def test_exact_factor_dataflow_off():
    """BSFM_BA_CHOL_DATAFLOW=0: systems <= 640 on the fused-step path, and the large path without its tail hand-over"""
    _child({"BSFM_BA_CHOL_DATAFLOW": "0"},
           [dict(n=n, s=s, dataflow=False) for n in (33, 97, 450, 640) for s in (0, -40)] +
           [dict(n=2560, s=s, dataflow=False, profile=True) for s in (0, 37)] +
           [dict(n=2560, pattern="band9", dataflow=False, profile=True)])


def test_exact_factor_tail_off():
    """BSFM_BA_CHOL_TAIL=0: every panel on the panel path, incl. a last panel 1 column wide (n = 2049)"""
    _child({"BSFM_BA_CHOL_TAIL": "0"}, [dict(n=n, s=s, tail_max=0, profile=True) for n in (2560, 2049) for s in (0, -40)])


def test_exact_factor_smallest_tail():
    """BSFM_BA_CHOL_TAIL=100 at n = 2113: the tail is 65 columns, the smallest one the hand-over takes"""
    _child({"BSFM_BA_CHOL_TAIL": "100"}, [dict(n=2113, s=s, tail_max=100, profile=True) for s in (0, 37)])


def test_exact_factor_refused_tail():
    """BSFM_BA_CHOL_TAIL=768 at n = 2689: chol_dataflow_factor refuses the 641-column remainder, the panel path goes on and
    hands over 385 columns one panel later"""
    _child({"BSFM_BA_CHOL_TAIL": "768"}, [dict(n=2689, s=s, tail_max=768, profile=True) for s in (0, -40)])


def test_exact_factor_lookahead_off():
    """BSFM_BA_CHOL_LOOKAHEAD=0: one trailing-update launch per panel, on the main stream"""
    _child({"BSFM_BA_CHOL_LOOKAHEAD": "0"},
           [dict(n=4500, s=s, lookahead=False, profile=True) for s in (0, -40)] +
           [dict(n=16897, pattern="band", lookahead=False, profile=True)])


# ---- why a factorisation failed -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,j", [(450, 200), (1100, 550), (1536, 200), (4500, 808), (2000, 1900)],
                         ids=["dataflow", "fused-step", "tile-kernel-step", "diagonal-kernel-sub-step", "large-path-tail"])
def test_zero_pivot_is_reported_as_a_pivot_failure(n, j):
    """L0_jj = 0: A is singular and the pivot of column j is exactly 0, with no rounding involved"""
    L0, A, x0, b = system(n, zero_pivots=(j,))
    rc, fail, *_ = factorise(A, b)
    assert (rc, fail) == (0, 1), (path_of(n), n, j, rc, fail)


# the placements of test_ba_gpu.py's test_axb_chol_reports_* tests: (n, seed, bad pivot)
REPORTS = [(300, 5, 150), (1100, 5, 550), (1350, 5, 675), (2000, 5, 1000), (1536, 7, 5), (1536, 7, 200), (1536, 7, 1530),
           (2000, 5, 1900), (450, 6, 3), (450, 6, 200), (450, 6, 449)]


@pytest.mark.parametrize("n,seed,where", REPORTS)
def test_negative_pivot_is_reported_as_a_pivot_failure(n, seed, where):
    """a negative diagonal entry fails with fail_code 1 (a non-positive pivot), never 2 (a lost dataflow word)"""
    A = spd(n, seed=seed)
    A[where, where] = -1.0
    rc, fail, *_ = factorise(A, np.ones(n))
    assert (rc, fail) == (0, 1), (path_of(n), n, where, rc, fail)


# ---- precision ------------------------------------------------------------------------------------------------------------
def well_conditioned(n, seed):
    """symmetric, diagonally dominant: off-diagonal uniform(-1, 1), a_ii = 1.5 r_i (r_i = the row's off-diagonal |sum|), so by
    Gershgorin every eigenvalue lies in [0.5 min r, 2.5 max r]: kappa <= 5 max r / min r"""
    rng = np.random.default_rng(seed)
    S = rng.uniform(-1.0, 1.0, (n, n))
    S = np.triu(S, 1)
    S = S + S.T
    r = np.abs(S).sum(axis=1)
    A = S + np.diag(1.5 * r)
    assert 5.0 * r.max() / r.min() <= 10.0
    return A


@pytest.mark.parametrize("n", [640, 1536, 4500])
def test_factor_precision_bound(n):
    """|A - fl(L L^T)| <= 4 (n + 1) u (|L||L|^T) entry by entry, u = 2^-53, on a well-conditioned random system.

    The constant: a Cholesky factorisation whose every entry is a sum of at most n products evaluated in fp64 has
    L L^T = A + dA with |dA| <= gamma_{n+1} |L||L|^T (Higham, Theorem 10.3).  The blocked paths also multiply by explicit
    inverses of the 32 x 32 and 256 x 256 diagonal blocks instead of solving with them; each such product adds at most
    gamma_{32} resp. gamma_{256} times |X||L_kk^-T||L_kk^T| to the panel X, and on these matrices (diagonally dominant, so
    |L_kk^-1||L_kk| stays O(1)) that is within another (n + 1) u |L||L|^T for n >= 640.  Forming fl(L L^T) in fp64 adds
    gamma_n |L||L|^T.  Together (n + 1) u (1 + 1 + 1) to first order, so 4 (n + 1) u leaves room for the second-order terms.
    A single step in fp32 leaves errors near 2^-24 |L_ik L_jk|, about 2^29 / (4 (n + 1)) > 10^4 times the bound."""
    A = well_conditioned(n, seed=n)
    b = np.ones(n)
    rc, fail, x, L, *_ = factorise(A, b)
    assert (rc, fail) == (1, 0)
    L = np.tril(L)
    u = 2.0 ** -53
    absL = np.abs(L)
    err = np.abs(A - L @ L.T)
    bound = 4.0 * (n + 1) * u * (absL @ absL.T)
    ratio = err / bound
    i, j = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio[i, j] <= 1.0, (path_of(n), n, "worst entry", (int(i), int(j)), float(err[i, j]), float(bound[i, j]),
                                _where(max(i, j), min(i, j), n))
