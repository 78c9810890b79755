"""Generates tests/golden/match_ties_golden.npz: the in-bundler matcher of the UNMODIFIED reference (MatchKeysExhaustive of
src/keys.cpp, test sqrt(d0 / d1) <= ratio, oracle/_ref/libref_keys.so) at ratio 1.0 and 0.75 on the tie-rich scenes of
tests/match_scenes.py and on all 110 ordered pairs of the kermit SIFT keys (tests/golden/kermit_match_golden.npz).

At ratio 1.0 (the symmetric pass of bundler --add_images) a query whose nearest distance is shared by several keys passes, so
which tied key is returned is part of the output.  The kd-tree returns the first key it visits; the GPU returns the smallest
caller index.  Stored per case: the nearest key of every query row (-1 = no match).  The scene descriptors are regenerated
from their seeds by the test, which checks them against the stored digests first.
   python tests/golden/make_match_ties_golden.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import loader  # noqa: E402
from tests import match_scenes  # noqa: E402

RATIOS = {"r100": 1.0, "r075": 0.75}


def tie_scenes():
    """(name, q, db) of the scenes recorded here"""
    return [(n, q, db) for n, q, db in match_scenes.all_scenes(seed=0)
            if n in ("sparse", "sparse_700", "near_duplicate", "two_equal_keys_db", "equal_norm_0.75")]


def kermit_pairs():
    g = np.load(os.path.join(HERE, "kermit_match_golden.npz"))
    descs = [g[f"desc{i}"] for i in range(int(g["num_images"]))]
    return [(f"kermit_{a}_{b}", descs[a], descs[b]) for a in range(len(descs)) for b in range(len(descs)) if a != b]


def digest(q, db):
    return np.frombuffer(hashlib.sha256(q.tobytes() + db.tobytes()).digest()[:8], np.uint64)[0]


def nearest_per_row(m, n1):
    nn = np.full(n1, -1, np.int32)
    nn[m[:, 0]] = m[:, 1]
    return nn


if __name__ == "__main__":
    out = {}
    for name, q, db in tie_scenes() + kermit_pairs():
        out[f"{name}_digest"] = np.array(digest(q, db))
        for tag, ratio in RATIOS.items():
            m = loader.keys_match_ref(q, db, None, False, ratio, exhaustive=True)
            out[f"{name}_{tag}"] = nearest_per_row(m, q.shape[0])
    np.savez_compressed(os.path.join(HERE, "match_ties_golden.npz"), **out)
    print("cases", len(out) // 3)
