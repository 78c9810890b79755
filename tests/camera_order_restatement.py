"""Restatement (CPU only, numpy / plain Python) of the camera order of large reduced camera systems (ba_order.cu:
bsfm_ba_camera_order), for tests/test_ba_camera_order.py.

The free cameras (j >= mcon) are the nodes of a graph with an edge for every off-diagonal block of S (a pair of cameras
that share a point).  Two orders are scored: the natural one and reverse Cuthill-McKee (George-Liu pseudo-peripheral start,
neighbours by ascending degree, ties by camera index, each connected component reversed in place, components in order of
their lowest camera).  The score of an order is the number of 128 x 128 tiles the large Cholesky's trailing update keeps
(ba_chol_large.cu: chol_syrk_dmma_kernel's row-block list), summed over its panels, from the block structure of L found
symbolically (elimination tree, children's structures merged into the parent)."""
import numpy as np

from tests.chol_exact_systems import PANEL, SLAB, TILE, SY_MAX_RB, LARGE_MIN, update_launches


def scene_block_keys(obs_pt, obs_cam, m, mcon=0):
    """the Schur pass's block keys j * m + k (j <= k, both >= mcon) of a visibility given as (point, camera) per observation
    (point-major, ascending camera within a point), ascending"""
    obs_pt, obs_cam = np.asarray(obs_pt, np.int64), np.asarray(obs_cam, np.int64)
    keep = obs_cam >= mcon
    obs_pt, obs_cam = obs_pt[keep], obs_cam[keep]
    ptr = np.concatenate([[0], np.cumsum(np.bincount(obs_pt, minlength=int(obs_pt.max()) + 1 if len(obs_pt) else 0))])
    keys = set()
    for i in range(len(ptr) - 1):
        cams = obs_cam[ptr[i]:ptr[i + 1]]
        for a in range(len(cams)):
            for b in range(a, len(cams)):
                keys.add(int(cams[a]) * m + int(cams[b]))
    return np.array(sorted(keys), np.uint32)


def circulant_block_keys(m, offsets):
    """block keys of the camera graph j ~ j + o (mod m) for o in offsets, diagonal included: the structure of
    synth.ba_scene's strided ring (camera j sees points together with j + step * t, t < views_per_point)"""
    keys = set()
    for j in range(m):
        keys.add(j * m + j)
        for o in offsets:
            k = (j + o) % m
            keys.add(min(j, k) * m + max(j, k))
    return np.array(sorted(keys), np.uint32)


def free_graph(keys, m, mcon):
    """adjacency lists (ascending) of the free cameras 0 .. m - mcon - 1 (camera j is node j - mcon)"""
    nf = m - mcon
    adj = [set() for _ in range(nf)]
    for key in np.asarray(keys, np.int64):
        j, k = int(key // m), int(key % m)
        if j != k and j >= mcon and k >= mcon:
            adj[j - mcon].add(k - mcon)
            adj[k - mcon].add(j - mcon)
    return [sorted(a) for a in adj]


def _levels(adj, root, mask):
    levels, seen = [[root]], {root}
    while True:
        nxt = []
        for v in levels[-1]:
            for u in adj[v]:
                if mask[u] and u not in seen:
                    seen.add(u)
                    nxt.append(u)
        if not nxt:
            return levels
        levels.append(nxt)


def rcm(adj):
    """reverse Cuthill-McKee order: order[q] = node at position q"""
    nf = len(adj)
    deg = [len(a) for a in adj]
    free = [True] * nf
    order = []
    for start in range(nf):
        if not free[start]:
            continue
        root = start
        levels = _levels(adj, root, free)
        while len(levels) > 1:      # George-Liu: a minimum-degree node of the last level, while the level structure deepens
            cand = min(levels[-1], key=lambda v: (deg[v], v))
            lv = _levels(adj, cand, free)
            root = cand
            if len(lv) <= len(levels):
                break
            levels = lv
        comp = [root]
        free[root] = False
        head = 0
        while head < len(comp):
            v = comp[head]
            head += 1
            nb = sorted((u for u in adj[v] if free[u]), key=lambda u: (deg[u], u))
            for u in nb:
                free[u] = False
            comp.extend(nb)
        order.extend(reversed(comp))
    return order


def l_structure(adj, pos):
    """block structure of L for the order pos (node -> position): struct[q] = positions > q of the nonzero blocks of column q"""
    nf = len(adj)
    node = [0] * nf
    for v, q in enumerate(pos):
        node[q] = v
    children = [[] for _ in range(nf)]
    struct = [None] * nf
    for q in range(nf):
        s = {pos[u] for u in adj[node[q]] if pos[u] > q}
        for c in children[q]:
            s |= struct[c]
        s.discard(q)
        struct[q] = s
        if s:
            children[min(s)].append(q)
    return struct


def slab_flags(struct, cnp):
    """per panel: the nonzero 64-row slabs (absolute slab index) below the diagonal block, right-hand-side row included"""
    nf = len(struct)
    n = nf * cnp
    nslab_all = (n + 1 + SLAB - 1) // SLAB
    flags = np.zeros(((n + PANEL - 1) // PANEL, nslab_all), np.int64)
    for p in range(flags.shape[0]):
        k0, k1 = p * PANEL, min(n, (p + 1) * PANEL)
        rows = set()
        for c in range(k0 // cnp, (k1 - 1) // cnp + 1):
            rows |= struct[c]
            if (c + 1) * cnp > k1:       # the camera straddles the panel's end: its own rows below k1 are nonzero
                rows.add(c)
        for J in rows:
            r0, r1 = max(J * cnp, k1), (J + 1) * cnp
            if r0 < r1:
                flags[p, r0 // SLAB:(r1 - 1) // SLAB + 1] = 1
        flags[p, n // SLAB] = 1          # the right-hand side
    return flags


def kept_tiles(flags, n):
    """tiles the trailing update keeps over all panels (the launches of chol_solve_large, look-ahead split included)"""
    tiles = 0
    for k1, cb, ce in update_launches(n):
        f = flags[k1 // PANEL - 1, k1 // SLAB:]
        nrows, nslab = n + 1, (n + 1 - k1 + SLAB - 1) // SLAB
        nrb, ncb, rb0 = -(-(nrows - cb) // TILE), -(-(ce - cb) // TILE), (cb - k1) // TILE
        kept = [rb for rb in range(nrb)
                if nrb > SY_MAX_RB or f[2 * (rb0 + rb)] or (2 * (rb0 + rb) + 1 < nslab and f[2 * (rb0 + rb) + 1])]
        for jj, j in enumerate(kept):
            if j < ncb:
                tiles += len(kept) - jj
    return tiles


def dense_tiles(n):
    return kept_tiles(np.ones(((n + PANEL - 1) // PANEL, (n + 1 + SLAB - 1) // SLAB), np.int64), n)


def score(adj, pos, cnp):
    return kept_tiles(slab_flags(l_structure(adj, pos), cnp), len(adj) * cnp)


def camera_order(keys, m, mcon, cnp):
    """-> (chosen, cam_pos, natural score, rcm score): what bsfm_ba_camera_order returns.  RCM is taken when it keeps at most
    three quarters of the natural order's tiles; systems of the small paths (n <= 1536) keep the natural order unscored."""
    adj = free_graph(keys, m, mcon)
    nf = len(adj)
    natural = list(range(nf))
    if nf * cnp <= LARGE_MIN:
        return 0, natural, 0, 0
    order = rcm(adj)
    pos = [0] * nf
    for q, v in enumerate(order):
        pos[v] = q
    s_nat, s_rcm = score(adj, natural, cnp), score(adj, pos, cnp)
    if 4 * s_rcm <= 3 * s_nat:
        return 1, pos, s_nat, s_rcm
    return 0, natural, s_nat, s_rcm
