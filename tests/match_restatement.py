"""Integer restatement of what the MATCH kernels decide for every query row (bundler_sfm_b200/csrc/match_kernels.cu).

`restate(q, db, ratio, mode, epilogue)` follows one (query image, database image) pair through the tensor-core path:
norm-sorted database, per-chunk bounds (bound epilogue, 64-column chunks) or exact chunk minima (exact epilogue, 32-column
chunks), the sequential row bookkeeping of `reduce_part`, the candidate test, `match_verify_kernel`'s match / reject / hard
split and `match_fullscan_kernel`.  Every quantity is an exact integer or the same double expression the kernel evaluates,
so the branch counts it returns are what the library must report, not approximations of it.

Among keys tied for the nearest distance the returned key is the one with the smallest caller index, on every kernel.
"""
import math

import numpy as np

NORM_PAD = 1 << 30
NORM_PAD_HALF = 1 << 29
INT_MAX = 2 ** 31 - 1
IMG_PAD = 256
BCHUNK = 64      # bound epilogue
CHUNK = 32       # exact epilogue
TC_NORM_CAP = 8192


def ratio_sq_host(ratio, mode):
    """P.ratio_sq of match_api.cu: test mode 1 inflates it so the pre-filters can never drop a row at the boundary"""
    return ratio * ratio if mode == 0 else ratio * ratio * (1.0 + 1e-9)


def ties_pass(ratio, mode):
    """P.ties_pass: does d0 == d1 > 0 pass the final test?"""
    return ratio * ratio > 1.0 if mode == 0 else ratio >= 1.0


def ratio_pass(d0, d1, ratio, mode):
    """ratio_pass of match_kernels.cuh on exact integers (d1 may be INT_MAX)"""
    if mode == 0:
        return float(d0) < (ratio * ratio) * float(d1)
    if d1 == 0:
        return False      # 0 / 0 = NaN
    return math.sqrt(float(d0) / float(d1)) <= ratio


def sqdist(q, db):
    q, db = q.astype(np.int64), db.astype(np.int64)
    return (q * q).sum(1)[:, None] + (db * db).sum(1)[None, :] - 2 * q @ db.T


def top2(d_row, key):
    """(d0, d1, index of the nearest) ordering by (distance, caller index); d1 = INT_MAX for a single key"""
    o = np.lexsort((key, d_row))
    d0 = int(d_row[o[0]])
    d1 = int(d_row[o[1]]) if len(o) > 1 else INT_MAX
    return d0, d1, int(o[0])


def passing_tie_rows(q, db, ratio, mode):
    """query rows whose nearest distance is shared by two keys and still passes the test: there the tie rule is visible"""
    if len(q) == 0 or len(db) < 2 or not ties_pass(ratio, mode):
        return np.zeros(0, np.int64)
    d = np.sort(sqdist(q, db), axis=1)
    return np.nonzero((d[:, 0] == d[:, 1]) & (d[:, 0] > 0))[0]


def restate(q, db, ratio, mode=0, epilogue="bound"):
    """-> (matches int32 [M, 2] in query order, counts dict).

    counts: candidates, hard (rows sent to the full scan), and the four outcomes verify_match, verify_reject, scan_match,
    scan_reject.  `epilogue` is "bound" (tc, tc_quad, tc_pair) or "exact" (tc_exact)."""
    counts = dict(candidates=0, hard=0, verify_match=0, verify_reject=0, scan_match=0, scan_reject=0)
    n1, n = len(q), len(db)
    if n1 == 0 or n == 0:
        return np.zeros((0, 2), np.int32), counts
    assert epilogue in ("bound", "exact")
    q64, db64 = q.astype(np.int64), db.astype(np.int64)
    nb = (db64 * db64).sum(1)
    order = np.argsort(nb, kind="stable")              # cub's stable segmented sort by squared norm
    npad = (n + IMG_PAD - 1) // IMG_PAD * IMG_PAD
    norms = np.full(npad, NORM_PAD, np.int64)
    norms[:n] = nb[order]
    perm = np.full(npad, -1, np.int64)
    perm[:n] = order
    dots = np.zeros((n1, npad), np.int64)
    dots[:, :n] = q64 @ db64[order].T
    na = (q64 * q64).sum(1)
    t = norms[None, :] - 2 * dots                      # t = |p|^2 - 2 q.p, padding columns included
    d_all = na[:, None] + t[:, :n]                     # exact distances in norm-sorted order
    rsq = ratio_sq_host(ratio, mode)
    ties = ties_pass(ratio, mode)

    M1 = np.full(n1, INT_MAX, np.int64)
    S2 = np.full(n1, INT_MAX, np.int64)
    BC = np.zeros(n1, np.int64)
    if epilogue == "bound":
        UBB = np.full(n1, INT_MAX, np.int64)
        UO = np.full(n1, INT_MAX, np.int64)
        for c in range(npad // BCHUNK):
            c0 = c * BCHUNK
            vmax = dots[:, c0:c0 + BCHUNK].max(1)
            lb = norms[c0] - 2 * vmax
            ub = norms[c0 + BCHUNK - 1] - 2 * vmax
            best = lb < M1
            S2 = np.where(best, M1, np.minimum(S2, lb))
            UO = np.minimum(UO, np.where(best, UBB, ub))
            UBB = np.where(best, ub, UBB)
            BC = np.where(best, c, BC)
            M1 = np.minimum(M1, lb)
        ubs = np.maximum(UBB, UO)
        d1u = np.where(ubs >= NORM_PAD_HALF, INT_MAX, na + ubs)
        cand = (na + M1).astype(np.float64) < rsq * d1u.astype(np.float64)
    else:
        for c in range(npad // CHUNK):
            cm = t[:, c * CHUNK:(c + 1) * CHUNK].min(1)
            hi = np.maximum(M1, cm)
            BC = np.where(cm < M1, c, BC)
            M1 = np.minimum(M1, cm)
            S2 = np.minimum(S2, hi)
        d1u = np.where(S2 >= NORM_PAD_HALF, INT_MAX, na + S2)
        cand = (na + M1).astype(np.float64) < rsq * d1u.astype(np.float64)

    width = BCHUNK if epilogue == "bound" else CHUNK
    out = []
    for r in np.nonzero(cand)[0]:
        counts["candidates"] += 1
        col0 = int(BC[r]) * width
        cols = slice(col0, min(col0 + width, n))
        m1, m2, mi = top2(d_all[r, cols], perm[cols])
        hard = match = False
        if epilogue == "exact":
            f5 = int(d1u[r])
            if ties and f5 == m1:
                hard = True
            else:
                match = ratio_pass(m1, min(f5, m2), ratio, mode)
        else:
            l2d = INT_MAX if S2[r] >= NORM_PAD_HALF else int(na[r] + S2[r])
            uod = INT_MAX if UO[r] >= NORM_PAD_HALF else int(na[r] + UO[r])
            if m1 > l2d or (ties and m1 == l2d):
                hard = True
            elif ratio_pass(m1, min(m2, l2d), ratio, mode):
                match = True
            elif ratio_pass(m1, min(m2, uod), ratio, mode):
                hard = True
        if match:
            counts["verify_match"] += 1
            out.append((r, int(perm[col0 + mi])))
        elif not hard:
            counts["verify_reject"] += 1
        else:
            counts["hard"] += 1
            f1, f2, fi = top2(d_all[r], perm[:n])
            if ratio_pass(f1, f2, ratio, mode):
                counts["scan_match"] += 1
                out.append((r, int(perm[fi])))
            else:
                counts["scan_reject"] += 1
    out.sort()
    return np.array(out, np.int32).reshape(-1, 2), counts


def library_epilogue(db_sizes, kernel):
    """the epilogue the library runs: bound unless forced to exact or some image of the run exceeds the norm staging buffer"""
    if kernel == "tc_exact":
        return "exact"
    padded = max((n + IMG_PAD - 1) // IMG_PAD * IMG_PAD for n in db_sizes)
    return "bound" if padded <= TC_NORM_CAP else "exact"
