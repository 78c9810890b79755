"""Seeded block-sparse SPD systems for the large Cholesky's zero-block skip (ba_chol_large.cu), shared by
tests/golden/make_chol_sparse_golden.py and tests/test_chol_sparse_gpu.py.

A system of size n has "cameras" of 9 rows (the last one may be shorter).  A = mu I + sum over coupling sets of a random
rank-3 PSD block over the rows of the set's cameras, b is random.  Everything is built from elementwise products and
additions in a fixed order (no BLAS), so the same seed gives the same bits on every machine.

Patterns (the coupling sets):
  ring       camera j with j + k step (mod m), k < 6: the benchmark scene's profile (banded, wrapping into dense last rows)
  band       camera j with j + 1, j + 2
  arrow      camera j with the last three cameras: only the last rows are dense
  blockdiag  every camera alone: below each panel only the straddling camera and the right-hand-side row are nonzero
"""
import numpy as np

CAM = 9
MU = 1.0

# (name, pattern, n): n = 1537, 2560, 3073 are the tile-edge and odd-pitch sizes of test_chol_trailing_gpu.py
CASES = [
    ("ring_4500", "ring", 4500),
    ("band_4005", "band", 4005),
    ("arrow_3600", "arrow", 3600),
    ("blockdiag_2560", "blockdiag", 2560),
    ("ring_1537", "ring", 1537),
    ("band_1537", "band", 1537),
    ("band_2560", "band", 2560),
    ("arrow_3073", "arrow", 3073),
    ("blockdiag_3073", "blockdiag", 3073),
]


def coupling_sets(pattern, m):
    if pattern == "ring":
        step = max(m // 6, 1)
        return [sorted({(j + k * step) % m for k in range(6)}) for j in range(m)]
    if pattern == "band":
        return [list(range(j, min(j + 3, m))) for j in range(m)]
    if pattern == "arrow":
        return [sorted({j, m - 3, m - 2, m - 1}) for j in range(m)]
    if pattern == "blockdiag":
        return [[j] for j in range(m)]
    raise ValueError(pattern)


def system(pattern, n, seed):
    """(A, b): A symmetric positive definite n x n with the pattern's block structure, b random"""
    rng = np.random.default_rng(seed)
    m = (n + CAM - 1) // CAM
    A = np.zeros((n, n))
    for cams in coupling_sets(pattern, m):
        idx = np.concatenate([np.arange(CAM * c, min(CAM * c + CAM, n)) for c in cams])
        g = rng.standard_normal((3, idx.size))
        P = g[0][:, None] * g[0][None, :]
        P = P + g[1][:, None] * g[1][None, :]
        P = P + g[2][:, None] * g[2][None, :]
        A[np.ix_(idx, idx)] += P
    A[np.arange(n), np.arange(n)] += MU
    b = rng.standard_normal(n)
    return A, b


def case_system(name):
    for nm, pattern, n in CASES:
        if nm == name:
            return system(pattern, n, seed=n)
    raise KeyError(name)
