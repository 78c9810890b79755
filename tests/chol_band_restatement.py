"""Restatement (CPU only, numpy / plain Python) of the band plan of large reduced camera systems (ba_order.cu:
chol_band_plan, bsfm_ba_chol_band_plan), and exactly representable systems with a given row envelope for
tests/test_chol_band_gpu.py.

Row i's first nonzero column first[i] is also that of the Cholesky factor.  In 32 x 32 tiles, block row rb starts at tile
env[rb] = min(first[rows of rb]) // 32, and the right-hand-side row (block row nbk) at 0.  Tile (rb, cb), env[rb] <= cb <= rb,
takes rank-32 updates at the steps max(env[rb], env[cb]) .. cb - 1 (cb - 2 on the diagonal); the plan fits a system of
4097 .. 24576 unknowns when at most 2 x workers tiles take updates at one step and the envelope's tiles fit the panel path's
256 x 256 inverse workspace."""
import numpy as np
import scipy.sparse as sp

from tests.chol_exact_systems import LIMIT, PANEL, _allowed_in_panel, bounds

SUB = 32
BAND_MIN_N, BAND_MAX_N = 4096, 24 * 1024      # systems of at most 4096 unknowns keep the panel path


def envelope(first, n):
    nbk = -(-n // SUB)
    first = np.minimum(np.asarray(first, np.int64), np.arange(n))
    return [int(first[rb * SUB:min(n, rb * SUB + SUB)].min()) // SUB for rb in range(nbk)] + [0]


def live_tiles(env):
    """(first step, last step, rb, cb) of every tile that takes an update from a worker"""
    nbk = len(env) - 1
    out = []
    for rb in range(nbk + 1):
        for cb in range(env[rb], min(rb, nbk - 1) + 1):
            kf, kl = max(env[rb], env[cb]), (cb - 2 if rb == cb else cb - 1)
            if kf <= kl:
                out.append((kf, kl, rb, cb))
    return out


def band_plan(first, n, workers):
    """-> (fits, env, tiles with the right-hand-side row, largest live set, worker CTAs used or 0): bsfm_ba_chol_band_plan"""
    env = envelope(first, n)
    nbk = len(env) - 1
    ntile = sum(rb - env[rb] + 1 for rb in range(nbk)) + nbk
    live = live_tiles(env)
    count = np.zeros(nbk + 1, np.int64)
    for kf, kl, _, _ in live:
        count[kf:kl + 1] += 1
    max_live = int(count.max())
    used = max(1, min(workers, max_live))
    fits = BAND_MIN_N < n <= BAND_MAX_N and max_live <= 2 * used and ntile <= -(-n // PANEL) * PANEL * PANEL // (SUB * SUB)
    return fits, env, ntile, max_live, (used if fits else 0)


def camera_first_cols(keys, m, mcon, cnp, pos):
    """first nonzero column of every row of S in the camera order pos (camera -> position)"""
    nf = m - mcon
    lo = list(pos)
    for key in np.asarray(keys, np.int64):
        j, k = int(key // m), int(key % m)
        if j >= mcon and k >= mcon:
            lo[j - mcon] = min(lo[j - mcon], pos[k - mcon])
            lo[k - mcon] = min(lo[k - mcon], pos[j - mcon])
    first = np.zeros(nf * cnp, np.int32)
    for v in range(nf):
        first[pos[v] * cnp:(pos[v] + 1) * cnp] = lo[v] * cnp
    return first


# ---- row envelopes ---------------------------------------------------------------------------------------------------
def tile_band_first(n, width):
    """every row block reaches `width` tiles left, its own included"""
    i = np.arange(n)
    return np.maximum(0, (i // SUB - width + 1) * SUB).astype(np.int32)


def camera_band_first(n, reach, cam=9, seed=0):
    """9-row cameras (straddling the tile edges) that reach back a random 0 .. reach cameras: a jagged, non-monotone envelope"""
    rng = np.random.default_rng(seed)
    m = -(-n // cam)
    back = rng.integers(0, reach + 1, m)
    q = np.arange(n) // cam
    return np.maximum(0, (q - back[q]) * cam).astype(np.int32)


# ---- exactly representable systems inside an envelope ------------------------------------------------------------------
def envelope_factor(first, seed=0, density=0.5, zero_pivots=()):
    """L0 (CSR int64): unit diagonal (0 at `zero_pivots`), off-diagonal entries in {-1, 0, +1} only at first[i] <= j < i,
    under the same in-panel rule as tests/chol_exact_systems.py (so every 32- and 256-aligned diagonal block's inverse is
    exactly I - N)"""
    n = len(first)
    first = np.asarray(first, np.int64)
    rng = np.random.default_rng(seed)
    chunks = []
    for r0 in range(0, n, 256):
        r1 = min(n, r0 + 256)
        c0 = int(first[r0:r1].min())
        i = np.arange(r0, r1)[:, None]
        j = np.arange(c0, r1)[None, :]
        ok = (j < i) & (j >= first[r0:r1][:, None]) & (((i // PANEL) != (j // PANEL)) | _allowed_in_panel(i, j))
        ok &= rng.random(ok.shape) < density
        v = np.where(ok, rng.integers(0, 2, ok.shape, dtype=np.int8) * 2 - 1, 0).astype(np.int8)
        chunks.append(sp.hstack([sp.csr_matrix((r1 - r0, c0), dtype=np.int64), sp.csr_matrix(v, dtype=np.int64),
                                 sp.csr_matrix((r1 - r0, n - r1), dtype=np.int64)], format="csr"))
    d = np.ones(n, np.int64)
    d[list(zero_pivots)] = 0
    L = (sp.vstack(chunks, format="csr") + sp.diags(d, format="csr", dtype=np.int64)).astype(np.int64).tocsr()
    L.eliminate_zeros()
    return L


def envelope_system(first, seed=0, density=0.5, zero_pivots=()):
    """(L0, A, x0, b) with A = L0 L0^T (its row envelope is `first`) and b = A x0, exact in float64"""
    L0 = envelope_factor(first, seed, density, zero_pivots)
    x0 = np.random.default_rng(seed + 1).integers(-3, 4, L0.shape[0]).astype(np.int64)
    bd = bounds(L0, x0)
    if max(bd.values()) >= LIMIT:
        raise ValueError(f"partial sums of this system reach 2^52: {bd}")
    A = (L0 @ L0.T).toarray().astype(np.float64)
    return L0, A, x0, A @ x0.astype(np.float64)
