"""CPU checks of the MATCH restatement (tests/match_restatement.py) and of the reference's behaviour on distance ties.

The restatement decides every query row the way the tensor-core kernels do, branch by branch, and must give the C port's
match list (oracle/match_oracle.c) on every adversarial scene.  tests/test_match_kernels.py then holds the GPU to the
restatement's branch counts."""
import os

import numpy as np
import pytest

from tests import match_restatement as R
from tests import match_scenes

GOLD = os.path.join(os.path.dirname(__file__), "golden", "match_ties_golden.npz")
RATIOS = [(0, 0.6), (0, 0.8), (0, 0.95), (0, 0.999), (1, 0.6), (1, 0.75), (1, 0.8), (1, 0.95), (1, 0.999), (1, 1.0)]
# kermit pairs (query image, database image) where MatchKeysExhaustive returns another of the keys tied for the nearest
# distance than the smallest caller index, at ratio 1.0
KERMIT_REF_TIE_DIFFERS = {(8, 2), (10, 2)}


@pytest.fixture(scope="module")
def scenes():
    return match_scenes.all_scenes(seed=0)


@pytest.mark.parametrize("epilogue", ["bound", "exact"])
def test_restatement_equals_port_on_every_scene(oracle, scenes, epilogue):
    for name, q, db in scenes:
        for mode, ratio in RATIOS:
            got, _ = R.restate(q, db, ratio, mode, epilogue)
            want = oracle.match_pair_port_test(q, db, ratio, mode)
            assert np.array_equal(got, want), (name, mode, ratio)


def test_scenes_reach_every_branch(scenes):
    """the scenes send rows down every path of the bound epilogue; tc_exact only defers rows with a cross-chunk tie"""
    tot = dict.fromkeys(("verify_match", "verify_reject", "scan_match", "scan_reject"), 0)
    ties_seen = 0
    for name, q, db in scenes:
        for mode, ratio in RATIOS:
            _, c = R.restate(q, db, ratio, mode, "bound")
            for k in tot:
                tot[k] += c[k]
            assert c["candidates"] == c["hard"] + c["verify_match"] + c["verify_reject"]
            _, ce = R.restate(q, db, ratio, mode, "exact")
            assert ce["hard"] == 0 or R.ties_pass(ratio, mode), (name, mode, ratio)
            ties_seen += len(R.passing_tie_rows(q, db, ratio, mode))
    assert all(v > 0 for v in tot.values()), tot
    assert ties_seen > 100


@pytest.mark.parametrize("num,den,ratio", [(9, 25, 0.6), (9, 16, 0.75)])
def test_boundary_scene_needs_mode1_inflation(oracle, num, den, ratio, monkeypatch):
    """den * d0 == num * d1 exactly, the second-nearest key in another chunk and tile: every row passes test mode 1 and only
    the 1e-9 inflation of ratio^2 keeps the candidate pre-filter from dropping it"""
    q, db = match_scenes.equal_norm(num, den)
    d = np.sort(R.sqdist(q, db), axis=1)
    assert np.all(den * d[:, 0] == num * d[:, 1]) and np.all(d[:, 2] > d[:, 1])
    want = oracle.match_pair_port_test(q, db, ratio, 1)
    assert want.shape[0] == q.shape[0] and oracle.match_pair_port_test(q, db, ratio, 0).shape[0] == 0
    got, c = R.restate(q, db, ratio, 1, "bound")
    assert np.array_equal(got, want) and c["verify_match"] == q.shape[0]
    monkeypatch.setattr(R, "ratio_sq_host", lambda r, m: r * r)
    assert R.restate(q, db, ratio, 1, "bound")[0].shape[0] == 0


def _tie_cases():
    from tests.golden import make_match_ties_golden as mk
    return mk, mk.tie_scenes() + mk.kermit_pairs()


def test_reference_ties_golden_vs_tie_rule(oracle):
    """the unmodified MatchKeysExhaustive equals the smallest-caller-index rule on every row without a passing tie; on a row
    with one it returns one of the tied nearest keys, and on the kermit keys a different one only on the listed pairs"""
    mk, cases = _tie_cases()
    g = np.load(GOLD)
    differs, tie_rows = set(), 0
    for name, q, db in cases:
        assert g[f"{name}_digest"] == mk.digest(q, db), name
        for tag, ratio in mk.RATIOS.items():
            ref = g[f"{name}_{tag}"]
            want = mk.nearest_per_row(oracle.match_pair_port_test(q, db, ratio, 1), q.shape[0])
            tied = R.passing_tie_rows(q, db, ratio, 1)
            tie_rows += len(tied)
            off = np.ones(q.shape[0], bool)
            off[tied] = False
            assert np.array_equal(ref[off], want[off]), (name, tag)
            if len(tied):
                d = R.sqdist(q[tied], db)
                assert np.all(d[np.arange(len(tied)), ref[tied]] == d.min(1)), (name, tag)
                if np.any(ref[tied] != want[tied]) and name.startswith("kermit_"):
                    differs.add(tuple(int(x) for x in name.split("_")[1:]))
    assert tie_rows > 100
    assert differs == KERMIT_REF_TIE_DIFFERS
