"""Exactly representable Cholesky systems (CPU only): A = L0 L0^T with an integer factor L0, for tests that compare every
entry the dense Cholesky paths compute (tests/test_chol_exact_gpu.py) with the exact answer.

L0 is unit lower triangular with off-diagonal entries in {-1, 0, +1}.  If every partial sum a path can form is an integer
below 2^52, every path computes exactly L0 (whatever its summation order, fusion or tensor-core accumulation order), and
exactly x0 from b = A x0.  `exact_system` refuses a system where one of the bounds below reaches 2^52.

Inside every 256-column diagonal panel block a nonzero (i, j), i > j, is allowed only where row i lies in an odd 16-row group
and column j in an even 16-column group (both counted from the panel's first column).  With N the strictly lower part of
any 32- or 256-aligned diagonal block, N^2 = 0, so the inverse of that block is exactly I - N: the reference for the
32 x 32 inverses (linv) and the 256 x 256 panel inverses (xinv) needs no arithmetic.  The potf2 still cancels real work: the
odd x odd quadrant of A's diagonal tiles is I + N N^T.

Below the diagonal panel blocks L0 is free: dense random entries, a band, or the block patterns of
tests/chol_sparse_systems.py (9-row "cameras" coupled as ring / band / arrowhead / block diagonal), which leave whole
64-row slabs of a panel at zero and so exercise the large path's zero-block skip.

A scaled variant multiplies L0 by 2^s: A by 4^s, pivots are 4^s, every inverse carries 2^-s, all exact in binary.

Restatement of the trailing update's executed FLOPs (ba_chol_large.cu: chol_solve_large, syrk_kept_elements) from the
factor's zero pattern, for bsfm_ba_chol_profile_read's fp64_flops."""
import numpy as np
import scipy.sparse as sp

from tests.chol_sparse_systems import CAM, coupling_sets

PANEL, SUB, GROUP, SLAB, TILE = 256, 32, 16, 64, 128
SY_MAX_RB = 128           # row blocks the trailing update's kept-tile list holds (ba_chol_large.cu)
TAIL_MAX = 640            # default BSFM_BA_CHOL_TAIL
DF_MAX_N, DF_MAX_NBK = 768, 20      # the dataflow kernel's own limits (ba_chol_large.cuh)
LARGE_MIN = 1536          # larger systems take the 256-column panel path
LIMIT = 1 << 52


def _allowed_in_panel(i, j):
    """(i, j) inside one diagonal panel block: row in an odd 16-row group, column in an even 16-column group"""
    return (((i % PANEL) // GROUP) % 2 == 1) & (((j % PANEL) // GROUP) % 2 == 0)


def factor(n, pattern="dense", seed=0, density=0.5, band=384, zero_pivots=()):
    """L0 as a scipy CSR matrix of int64: unit diagonal (0 at `zero_pivots`), off-diagonal entries in {-1, 0, +1}.
    pattern: "dense" (every entry below the diagonal panel blocks may be nonzero), "band" (entries with i - j <= `band`),
    or a pattern of tests/chol_sparse_systems.py ("ring", "band9", "arrow", "blockdiag": allowed where the 9-row cameras
    of i and j are coupled)."""
    rng = np.random.default_rng(seed)
    pairs = None
    if pattern not in ("dense", "band"):
        m = (n + CAM - 1) // CAM
        pairs = np.zeros((m, m), bool)
        for s in coupling_sets("band" if pattern == "band9" else pattern, m):
            pairs[np.ix_(s, s)] = True
    chunks = []
    for r0 in range(0, n, 256):          # 256-row chunks: dense cases never hold an n x n boolean array
        r1 = min(n, r0 + 256)
        c0 = max(0, r0 - band) if pattern == "band" else 0
        i = np.arange(r0, r1)[:, None]
        j = np.arange(c0, r1)[None, :]
        ok = (j < i) & (((i // PANEL) != (j // PANEL)) | _allowed_in_panel(i, j))
        if pattern == "band":
            ok &= i - j <= band
        if pairs is not None:
            ok &= pairs[i // CAM, j // CAM]
        ok &= rng.random(ok.shape) < density
        v = np.where(ok, rng.integers(0, 2, ok.shape, dtype=np.int8) * 2 - 1, 0).astype(np.int8)
        chunk = sp.csr_matrix(v, dtype=np.int64)
        chunks.append(sp.hstack([sp.csr_matrix((r1 - r0, c0), dtype=np.int64), chunk,
                                 sp.csr_matrix((r1 - r0, n - r1), dtype=np.int64)], format="csr"))
    d = np.ones(n, np.int64)
    d[list(zero_pivots)] = 0
    L = (sp.vstack(chunks, format="csr") + sp.diags(d, format="csr", dtype=np.int64)).astype(np.int64).tocsr()
    L.eliminate_zeros()
    return L


def block_inverse_ref(L0, k0, size):
    """the exact inverse I - N of the diagonal block [k0, k0 + size) of a unit L0 (int64, dense)"""
    B = L0[k0:k0 + size, k0:k0 + size].toarray()
    return 2 * np.eye(B.shape[0], dtype=np.int64) - B


def bounds(L0, x0):
    """upper bounds (int64) of every partial sum the paths form, by kind:
      update     |L0||L0|^T            (the trailing updates, potf2, the right-hand-side row's forward substitution)
      rhs        |L0||L0|^T |x0|       (b and the right-hand-side row as it is updated)
      panel      |L0_below||L0_kk|^T|Z|^T per panel  (X Z^T products of the panel solves, Z = L0_kk^-1 = I - N)
      backsolve  |xinv||y| and |L0|^T|x0|  (the substitutions, y = L0^T x0)
    Entries are in {-1, 0, 1}, so (|L0||L0|^T)_ij <= min(r_i, r_j), r = nonzeros per row."""
    n = L0.shape[0]
    A1 = abs(L0).astype(np.int64)
    r = np.asarray(A1.sum(axis=1)).ravel()
    ax = np.abs(x0).astype(np.int64)
    out = {"update": int(r.max()), "rhs": int((A1 @ (A1.T @ ax)).max())}
    y = np.abs(L0.T @ x0.astype(np.int64))
    panel, back = 0, int((A1.T @ ax).max())
    for k0 in range(0, n, PANEL):
        k1 = min(n, k0 + PANEL)
        Lkk = A1[k0:k1, k0:k1].toarray()
        Z = np.abs(block_inverse_ref(L0, k0, k1 - k0))
        M = Lkk.T @ Z.T                                # (|L_kk|^T |Z|^T): its largest entry times the row's count below
        below = A1[k1:, k0:k1]
        if below.shape[0]:
            panel = max(panel, int(np.asarray(below.sum(axis=1)).max()) * int(M.max()))
        back = max(back, int((Z.T @ y[k0:k1]).max()))
    out["panel"], out["backsolve"] = panel, back
    return out


def exact_system(n, pattern="dense", seed=0, density=0.5, band=384, zero_pivots=()):
    """(L0 CSR int64, A float64 dense, x0 int64, b float64) with A = L0 L0^T and b = A x0 exact in float64.
    Raises ValueError when a partial-sum bound reaches 2^52."""
    L0 = factor(n, pattern, seed, density, band, zero_pivots)
    x0 = np.random.default_rng(seed + 1).integers(-3, 4, n).astype(np.int64)
    bd = bounds(L0, x0)
    if max(bd.values()) >= LIMIT:
        raise ValueError(f"partial sums of this system reach 2^52: {bd}")
    if pattern == "dense":       # BLAS: every partial sum is an integer below 2^53, so the product is exact in any order
        Ld = L0.toarray().astype(np.float64)
        A = Ld @ Ld.T
    else:
        A = (L0 @ L0.T).toarray().astype(np.float64)
    b = A @ x0.astype(np.float64)
    return L0, A, x0, b


def scaled(A, b, s):
    """A, b of the system with factor 2^s L0 and the same x0: A 4^s, b 4^s"""
    return np.ldexp(A, 2 * s), np.ldexp(b, 2 * s)


# ---- executed FLOPs of the trailing update (bsfm_ba_chol_profile_read) ------------------------------------------------
def tail_taken(n, kk, dataflow=True):
    """chol_dataflow_factor accepts the remaining n - kk columns (at most 20 blocks of 32 and DF_MAX_N rows)"""
    m = n - kk
    return dataflow and (m + SUB - 1) // SUB <= DF_MAX_NBK and m <= DF_MAX_N and (m + SUB - 1) // SUB >= 2


def update_launches(n, lookahead=True, tail_max=TAIL_MAX, dataflow=True):
    """the trailing-update launches (k1, cb, ce) of chol_solve_large, k1 = first row of the panel image"""
    def tail_fits(kk):
        return 0 < kk < n and 2 * SUB < n - kk <= tail_max
    out, diag_done = [], False
    for k0 in range(0, n, PANEL):
        k1 = min(n, k0 + PANEL)
        if not diag_done and tail_fits(k0) and tail_taken(n, k0, dataflow):
            break
        diag_done = False
        if k1 < n:
            k2 = min(n, k1 + PANEL)
            if lookahead and k2 < n and not tail_fits(k1):
                out += [(k1, k1, k2), (k1, k2, n)]
                diag_done = True
            else:
                out.append((k1, k1, n))
    return out


def kept_elements(flags, n, k1, cb, ce):
    """syrk_kept_elements: flags[s] = the bits (1 nonzero, 2 non-finite) of the panel solve's 64-row slab s (rows k1 + 64 s ..,
    right-hand-side row n included)"""
    nrows = n + 1
    nslab = len(flags)
    nrb, ncb, rb0 = -(-(nrows - cb) // TILE), -(-(ce - cb) // TILE), (cb - k1) // TILE
    f = [flags[2 * (rb0 + rb)] | (flags[2 * (rb0 + rb) + 1] if 2 * (rb0 + rb) + 1 < nslab else 0) for rb in range(nrb)]
    if nrb > SY_MAX_RB or any(v & 2 for v in f):
        kept = list(range(nrb))
    else:
        kept = [rb for rb in range(nrb) if f[rb]]
    el = 0
    for j in (j for j in kept if j < ncb):
        c0, c1 = cb + TILE * j, min(cb + TILE * (j + 1), ce)
        for i in (i for i in kept if i >= j):
            r0, r1 = cb + TILE * i, min(cb + TILE * (i + 1), nrows)
            if r0 >= c1:
                el += (r1 - r0) * (c1 - c0)
            else:
                c = np.arange(c0, c1)
                el += int(np.maximum(0, r1 - np.maximum(r0, c)).sum())
    return el


def slab_flags(L0, y):
    """per panel p: the nonzero bits of the 64-row slabs below it (rows p*256 + 256 + 64 s ..), from the pattern of L0 and of
    the right-hand-side row y (= L0^T x0, the forward substitution's result)"""
    n = L0.shape[0]
    nrows = n + 1
    nz = np.zeros(((n + PANEL - 1) // PANEL, (nrows + SLAB - 1) // SLAB), np.int64)
    C = L0.tocoo()
    keep = C.row >= (C.col // PANEL + 1) * PANEL
    nz[C.col[keep] // PANEL, C.row[keep] // SLAB] = 1
    j = np.nonzero(y)[0]
    nz[j // PANEL, n // SLAB] = 1
    return nz


def executed_flops(n, flags, lookahead=True, tail_max=TAIL_MAX, dataflow=True):
    """fp64_flops of one solve of size n: 2 x 256 x the kept lower-triangle elements of every trailing-update launch;
    flags as slab_flags returns them"""
    el = 0
    for k1, cb, ce in update_launches(n, lookahead, tail_max, dataflow):
        el += kept_elements(list(flags[k1 // PANEL - 1, k1 // SLAB:]), n, k1, cb, ce)
    return 2.0 * PANEL * el
