"""CPU tests: the premises of tests/test_chol_exact_gpu.py, so that a failure there can only mean a kernel is wrong.
  - A = L0 L0^T is exact in float64, and every partial-sum bound of every system the GPU tests use is below 2^52
  - the inverse of every diagonal 32- and 256-block is I - N
  - LAPACK's Cholesky returns L0 bit for bit
  - the tensor-core potf2's reciprocal square root (ba_chol_potf2.cuh: rsqrt_pos_normal), emulated in exact rational
    arithmetic, returns exactly 2^-k on 4^k for seeds across its whole error band, so the scaled systems stay exact
  - the restatement of the trailing update's executed FLOPs, on hand-worked cases and against test_chol_sparse_gpu.py's"""
import struct
from fractions import Fraction

import numpy as np
import pytest
from scipy.linalg import solve_triangular

from tests.chol_exact_systems import (LIMIT, PANEL, SUB, block_inverse_ref, bounds, exact_system, executed_flops, factor,
                                      kept_elements, scaled, slab_flags, update_launches)
from tests.test_chol_exact_gpu import SIZES, SPARSE
from tests.test_chol_sparse_gpu import _executed_flops


@pytest.mark.parametrize("n,pattern", [(300, "dense"), (1800, "dense"), (1537, "ring"), (2560, "blockdiag"), (2000, "band")])
def test_product_is_exact(n, pattern):
    L0, A, x0, b = exact_system(n, pattern, seed=n)
    Ai = (L0 @ L0.T).toarray()
    assert np.array_equal(A, Ai.astype(np.float64)) and np.array_equal(A.astype(np.int64), Ai)
    assert np.array_equal(b.astype(np.int64), Ai @ x0)
    As, bs = scaled(A, b, -40)
    assert np.array_equal(As, A * 2.0 ** -80) and np.array_equal(np.ldexp(As, 80), A)


@pytest.mark.parametrize("n,pattern", [(c[0], "dense") for c in SIZES] + [(n, p) for p, n in SPARSE] + [(16897, "band")])
def test_partial_sums_stay_below_2_52(n, pattern):
    L0 = factor(n, pattern, seed=n)
    x0 = np.random.default_rng(n + 1).integers(-3, 4, n)
    bd = bounds(L0, x0)
    assert max(bd.values()) < LIMIT, bd


def test_bounds_bound_the_exact_partial_sums():
    n = 700
    L0, A, x0, b = exact_system(n, seed=3)
    A1 = np.abs(L0.toarray())
    bd = bounds(L0, x0)
    assert (A1 @ A1.T).max() <= bd["update"]
    assert (A1 @ (A1.T @ np.abs(x0))).max() <= bd["rhs"]
    y = L0.T @ x0
    assert np.abs(y).max() <= bd["backsolve"] and (A1.T @ np.abs(x0)).max() <= bd["backsolve"]


@pytest.mark.parametrize("n,pattern", [(1, "dense"), (65, "dense"), (1249, "dense"), (2689, "dense"), (3073, "arrow"), (16897, "band")])
def test_diagonal_block_inverses_are_I_minus_N(n, pattern):
    L0 = factor(n, pattern, seed=n)
    for size in (SUB, PANEL):
        for k0 in range(0, n, size):
            w = min(size, n - k0)
            B = L0[k0:k0 + w, k0:k0 + w].toarray()
            Z = block_inverse_ref(L0, k0, w)
            assert np.array_equal(B @ Z, np.eye(w, dtype=np.int64)), (size, k0)
            assert np.array_equal(Z @ B, np.eye(w, dtype=np.int64)), (size, k0)
            N = B - np.eye(w, dtype=np.int64)
            assert not (N @ N).any()
            assert set(np.unique(B)) <= {-1, 0, 1}


@pytest.mark.parametrize("n", [9, 97, 640, 1100, 1547])
@pytest.mark.parametrize("s", [0, -40, 37])
def test_lapack_cholesky_returns_L0(n, s):
    L0, A, x0, b = exact_system(n, seed=n)
    A, b = scaled(A, b, s)
    L = np.linalg.cholesky(A)
    assert np.array_equal(L, np.ldexp(L0.toarray().astype(np.float64), s))
    y = solve_triangular(L, b, lower=True)
    assert np.array_equal(solve_triangular(L.T, y, lower=False), x0.astype(np.float64))


# ---- rsqrt_pos_normal (ba_chol_potf2.cuh) in exact rational arithmetic ------------------------------------------------------
def _rn(q):
    """round a rational to the nearest double, ties to even (int / int true division in Python is correctly rounded)"""
    return q.numerator / q.denominator


def rsqrt_pos_normal(d, y0):
    """t = d y0; e = fma(-t, y0, 1); p = fma(0.375, e, 0.5); u = y0 e; return fma(u, p, y0) -- each step rounded once"""
    F = Fraction
    t = _rn(F(d) * F(y0))
    e = _rn(-F(t) * F(y0) + 1)
    p = _rn(F(0.375) * F(e) + F(0.5))
    u = _rn(F(y0) * F(e))
    return _rn(F(u) * F(p) + F(y0))


def _high_word_only(y):
    hi = struct.unpack("<Q", struct.pack("<d", y))[0] & 0xFFFFFFFF00000000
    return struct.unpack("<d", struct.pack("<Q", hi))[0]


def test_rsqrt_is_exact_on_powers_of_four():
    """the seed of rsqrt.approx.ftz.f64 reads the high word only and is within 2^-20.5 relative: seeds spread over that whole
    band (and truncated to their high word like the hardware's) all give exactly 2^-k for pivots 4^k, k in [-60, 60]"""
    band = 2.0 ** -20.5
    tried = 0
    for k in range(-60, 61):
        d, want = 4.0 ** k, 2.0 ** -k
        for f in np.linspace(-band, band, 61):
            y0 = _high_word_only(want * (1.0 + f))
            assert rsqrt_pos_normal(d, y0) == want, (k, f)
            tried += 1
    assert tried == 121 * 61


# ---- the FLOP restatement -------------------------------------------------------------------------------------------------
def test_update_launches_hand_worked():
    # n = 1537: look-ahead splits while the next panel's remainder is > 640; the tail takes over at 1024 (513 columns)
    assert update_launches(1537) == [(256, 256, 512), (256, 512, 1537), (512, 512, 768), (512, 768, 1537),
                                     (768, 768, 1024), (768, 1024, 1537), (1024, 1024, 1537)]
    assert update_launches(1537, lookahead=False) == [(256, 256, 1537), (512, 512, 1537), (768, 768, 1537), (1024, 1024, 1537)]
    # tail off: every panel with columns right of it has an update; n = 2049 ends on a 1-column panel
    assert update_launches(2049, lookahead=False, tail_max=0) == [(k, k, 2049) for k in range(256, 2049, 256)]
    # a 641-column remainder is refused by the dataflow kernel: the panel path goes on, the tail takes 385 columns
    assert update_launches(2689, lookahead=False, tail_max=768) == [(k, k, 2689) for k in range(256, 2305, 256)]
    # by default the 641 columns are more than the tail takes: the same panels, but with the look-ahead panel 7's update
    # (k1 = 2048) is split, while with BSFM_BA_CHOL_TAIL=768 the next remainder "fits" and it is one launch
    assert update_launches(2689, lookahead=False) == [(k, k, 2689) for k in range(256, 2305, 256)]
    split = [(k, k, k + 256) for k in range(256, 2049, 256)]
    rest = [(k, k + 256, 2689) for k in range(256, 2049, 256)]
    assert update_launches(2689) == [v for pair in zip(split, rest) for v in pair] + [(2304, 2304, 2689)]
    assert update_launches(2689, tail_max=768) == update_launches(2689)[:14] + [(2048, 2048, 2689), (2304, 2304, 2689)]
    # n = 2688: the tail takes the last 640 columns, right after panel 7's unsplit update
    assert update_launches(2688) == [v for k in range(256, 2049 - 256, 256) for v in ((k, k, k + 256), (k, k + 256, 2688))] + \
        [(2048, 2048, 2688)]
    # dataflow off: no tail at all
    assert update_launches(2560, lookahead=False, dataflow=False) == [(k, k, 2560) for k in range(256, 2560, 256)]


def test_kept_elements_hand_worked():
    # n = 511, one update of rows 256..511 (row 511 = right-hand side) x columns 256..510: two 128-row blocks, 4 slabs
    dense = 32895            # sum_{c=256}^{510} (512 - c)
    assert kept_elements([1, 1, 1, 1], 511, 256, 256, 511) == dense
    assert kept_elements([0, 0, 1, 0], 511, 256, 256, 511) == 8255          # row block 1 only: its diagonal tile
    assert kept_elements([1, 0, 0, 0], 511, 256, 256, 511) == 8256          # row block 0 only
    assert kept_elements([1, 0, 0, 1], 511, 256, 256, 511) == dense
    assert kept_elements([2, 0, 0, 0], 511, 256, 256, 511) == dense         # a non-finite value keeps every tile
    assert kept_elements([0, 0, 0, 0], 511, 256, 256, 511) == 0
    # more than 128 row blocks in one launch keep every tile, whatever the flags
    n = 16897
    k1 = 256
    nslab = -(-(n + 1 - k1) // 64)
    flags = [0] * nslab
    flags[5] = 1
    cb, ce = 256, 512
    full = kept_elements([1] * nslab, n, k1, cb, ce)
    assert kept_elements(flags, n, k1, cb, ce) == full == sum(n + 1 - c for c in range(256, 512))
    cb, ce = 768, n                # 127 row blocks: the list
    assert kept_elements([0] * nslab, n, 512, cb, ce) == 0


@pytest.mark.parametrize("pattern,n", [("ring", 4500), ("band9", 4005), ("arrow", 3600), ("blockdiag", 2560), ("dense", 2560)])
def test_flop_restatement_agrees_with_the_one_launch_per_panel_model(pattern, n):
    """with no launch above 128 row blocks the look-ahead split executes the same tiles as one launch per panel"""
    L0 = factor(n, pattern, seed=n)
    x0 = np.random.default_rng(n + 1).integers(-3, 4, n)
    y = L0.T @ x0
    nonzero = np.vstack([L0.toarray() != 0, (y != 0)[None, :]])
    fl = slab_flags(L0, y)
    want = _executed_flops(nonzero, n)
    assert executed_flops(n, fl) == want
    assert executed_flops(n, fl, lookahead=False) == want
