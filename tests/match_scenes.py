"""Adversarial descriptor sets for the MATCH kernels, deterministic given a seed.

Each generator returns (query keys, database keys) as uint8 [n, 128].  They aim at the places where the bound epilogue's
decisions are fragile: wide norm spans inside a chunk, exact distance ties (also across chunk and tile boundaries),
near-duplicate keys of different norms, and rows sitting exactly on the ratio-test boundary."""
import numpy as np


def norm_spread(n1=200, n2=300, seed=0):
    """uniform keys, each scaled by its own random factor: a chunk's norms span a wide range, so its bounds are loose"""
    rng = np.random.default_rng(seed)
    q = (rng.integers(0, 256, (n1, 128)) * rng.uniform(0, 1, (n1, 1))).astype(np.uint8)
    db = (rng.integers(0, 256, (n2, 128)) * rng.uniform(0, 1, (n2, 1))).astype(np.uint8)
    return q, db


def sparse(n1=200, n2=300, seed=0):
    """1-5 non-zero bytes of value 1-3 per key: many exact distance ties"""
    rng = np.random.default_rng(seed)
    out = []
    for n in (n1, n2):
        a = np.zeros((n, 128), np.uint8)
        for r in range(n):
            idx = rng.choice(128, rng.integers(1, 6), replace=False)
            a[r, idx] = rng.integers(1, 4, len(idx))
        out.append(a)
    return out[0], out[1]


def near_duplicate(n1=300, seed=0):
    """every query plus two copies perturbed by -2..2 per byte in the database; the copies' norms differ"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (n1, 128)).astype(np.int64)
    copies = [np.clip(base + rng.integers(-2, 3, base.shape), 0, 255) for _ in range(2)]
    return base.astype(np.uint8), np.concatenate(copies).astype(np.uint8)


def _boundary_constants(num, den):
    """smallest (a, b, c, e) with a > b > 0, c > e > 0, den * d0 == num * d1 for the distances of equal_norm, and every
    other key of that scene strictly farther than d1"""
    for s in range(4, 400):
        for a in range(2, min(s, 256)):
            for c in range(2, min(s - a, 256)):
                e_b = s - a - c
                for b in range(1, min(a, e_b)):
                    e = e_b - b
                    if not (0 < e < c) or c * (a - b) >= e * a:
                        continue
                    K = a * a + b * b + c * c + e * e
                    d0, d1 = K - 2 * (c * a + e * b), K - 2 * (c * b + e * a)
                    if d0 > 0 and den * d0 == num * d1:
                        return a, b, c, e
    raise ValueError("no constants")


def equal_norm(ratio_num=9, ratio_den=25, n1=16, n2=600, near_pos=5, second_off=300, seed=0):
    """database keys are byte permutations of one vector (a at one position, b at another), so every key has the same norm,
    chunk bounds are exact and the pre-filters see the true d0 and d1.  Query r (c at position s_r, e at t_r) is nearest to
    its key (a at s_r, b at t_r) and second nearest to (b at s_r, a at t_r), with  ratio_den * d0 == ratio_num * d1:  the
    squared ratio sits exactly on the boundary.  The two keys lie `second_off` rows apart (another 64-column chunk and
    another 256-row tile); all other keys are strictly farther."""
    a, b, c, e = _boundary_constants(ratio_num, ratio_den)
    rng = np.random.default_rng(seed)
    pos = rng.permutation(128)[:2 * n1].reshape(n1, 2)      # disjoint position pairs: no key is special for two queries
    q = np.zeros((n1, 128), np.uint8)
    db = np.zeros((n2, 128), np.uint8)
    special = {}
    for r, (s, t) in enumerate(pos):
        q[r, s], q[r, t] = c, e
        special[near_pos + r] = (s, t)
        special[near_pos + second_off + r] = (t, s)
    used = {tuple(sorted(p)) for p in pos.tolist()}
    for k in range(n2):
        if k in special:
            i, j = special[k]
        else:
            while True:     # a filler shares at most one position with any query pair
                i, j = (int(x) for x in rng.choice(128, 2, replace=False))
                if tuple(sorted((i, j))) not in used:
                    break
        db[k, i], db[k, j] = a, b
    return q, db


def small_cases(seed=0):
    """zero queries, all-255 keys, one- and two-key databases -> list of (name, q, db)"""
    rng = np.random.default_rng(seed)
    rnd = rng.integers(0, 256, (40, 128)).astype(np.uint8)
    zeros = np.zeros((5, 128), np.uint8)
    full = np.full((3, 128), 255, np.uint8)
    mixed = np.concatenate([full, zeros, rnd[:10]])
    return [("zero_queries", zeros, rnd),
            ("all_255_db", rnd, np.concatenate([full, rnd[:7]])),
            ("all_255_queries", np.concatenate([full, rnd[:5]]), mixed),
            ("single_key_db", rnd, rnd[7:8]),
            ("single_zero_key_db", np.concatenate([zeros, rnd[:5]]), zeros[:1]),
            ("two_key_db", rnd, rnd[3:5]),
            ("two_equal_keys_db", np.concatenate([rnd[:5], zeros]), np.stack([rnd[9], rnd[9]])),
            ("two_zero_keys_db", np.concatenate([zeros, rnd[:5]]), zeros[:2])]


def all_scenes(seed=0):
    """every scene of the suite -> list of (name, q, db)"""
    s = [("norm_spread", *norm_spread(200, 300, seed)),
         ("norm_spread_513", *norm_spread(150, 513, seed + 1)),
         ("sparse", *sparse(200, 300, seed)),
         ("sparse_700", *sparse(200, 700, seed + 1)),
         ("near_duplicate", *near_duplicate(300, seed)),
         ("equal_norm_0.6", *equal_norm(9, 25, seed=seed)),
         ("equal_norm_0.75", *equal_norm(9, 16, seed=seed))]
    return s + small_cases(seed)
