"""The loop of BundlerApp::RunSFM_SBA restated (tests/outlier_loop_restatement.py): its compaction rule on hand-made CRS
arrays, its control flow over stub solvers, and, where oracle/_ref is built, the reference behind it against the committed
tests/golden/outlier_loop_golden.npz."""
import os

import numpy as np
import pytest

from bundler_sfm_b200 import synth
from tests import outlier_loop_restatement as rs
from tests import outlier_loop_scenes as scenes

GOLD = os.path.join(os.path.dirname(__file__), "golden", "outlier_loop_golden.npz")

PTR = [0, 0, 2, 2, 2, 5, 6, 6]          # 7 points: empty first, adjacent empties in the middle, empty last
CAM = [0, 3, 1, 2, 4, 0]
PROJ = np.arange(12, dtype=np.float64).reshape(6, 2)


@pytest.mark.parametrize("keep,want_ptr,want_obs,want_orig", [
    ([0, 1, 0, 0, 1, 1, 0], [0, 2, 5, 6], [0, 1, 2, 3, 4, 5], [1, 4, 5]),      # exactly the points with views
    ([1, 1, 1, 1, 1, 1, 1], PTR, [0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5, 6]),   # none removed: empties stay empty rows
    ([0, 0, 0, 0, 0, 0, 0], [0], [], []),                                      # every point removed
    ([0, 1, 0, 0, 0, 1, 0], [0, 2, 3], [0, 1, 5], [1, 5]),                     # a point with views removed: all its views go
    ([0, 0, 0, 0, 1, 0, 0], [0, 3], [2, 3, 4], [4]),
])
def test_compaction_rule(keep, want_ptr, want_obs, want_orig):
    ptr, cam, proj, orig = rs.compact_crs(PTR, CAM, PROJ, keep)
    assert ptr.tolist() == list(want_ptr) and orig.tolist() == list(want_orig)
    assert cam.tolist() == [CAM[o] for o in want_obs]
    assert np.array_equal(proj, PROJ[want_obs].reshape(-1, 2))


def stub_scene(n=12):
    ptr = np.arange(n + 1, dtype=np.int32)
    ptr[3:] -= 1                                    # point 2 has no view on entry
    return {"vis_ptr": ptr, "vis_cam": np.zeros(n - 1, np.int32), "projections": np.zeros((n - 1, 2)),
            "R": np.eye(3).reshape(1, 9), "c": np.zeros((1, 3)), "f": np.ones(1), "k": np.zeros((1, 2)),
            "pts": np.arange(3 * n, dtype=np.float64).reshape(n, 3)}


def stub_loop(flag_per_round, seen, **kw):
    """solve adds 100 to every point and records the constraint rows it was given; the pass of round r flags the round's
    first flag_per_round[r] unprotected points"""
    scene = stub_scene()

    def solve(s, pc):
        seen.append((len(s["pts"]), None if pc is None else pc.copy()))
        return {**{k: s[k] for k in rs.CAMERA_KEYS}, "pts": s["pts"] + 100.0, "info": np.zeros(10)}

    def outlier_pass(s, prot):
        r = len(seen) - 1
        free = [q for q in range(len(s["pts"])) if prot is None or not prot[q]]
        out = free[:flag_per_round[r]]
        return {"outliers": out, "errors": [50.0 + q for q in out], "stats": np.zeros((1, 5)), "global_mean": 1.0 + r}

    return rs.run_loop(scene, solve, outlier_pass, **kw)


def test_loop_stops_when_a_round_removes_at_most_min_outliers_and_still_removes_them():
    seen = []
    out = stub_loop([3, 2, 9], seen, min_outliers=2, min_points=1)
    assert out["count"] == 2 and [s[0] for s in seen] == [11, 8]
    assert out["pt_round"].tolist() == [0, 0, -2, 0, 1, 1, -1, -1, -1, -1, -1, -1]
    assert out["pt_error"][:6].tolist() == [50.0, 51.0, 0.0, 52.0, 50.0, 51.0]     # errors follow the round's numbering
    assert out["mean_error"] == 2.0
    # write-back: a point removed in round 0 was solved once, a survivor twice, the empty point never
    assert out["pts"][0, 0] == 100.0 and out["pts"][4, 0] == 12.0 + 200.0 and out["pts"][2, 0] == 6.0


def test_loop_ends_on_too_few_points_counted_on_the_original_number():
    seen = []
    out = stub_loop([5, 5], seen, min_outliers=2, min_points=8)
    assert out["count"] == 1 and out["mean_error"] == rs.DBL_MAX           # 12 - 5 < 8, although only 6 points had remained
    seen = []
    assert stub_loop([5, 5], seen, min_outliers=2, min_points=13)["count"] == 0


def test_loop_without_removal_runs_one_round():
    seen = []
    out = stub_loop([5, 5], seen, remove_outliers=0, min_outliers=2, min_points=1)
    assert out["count"] == 1 and np.all(out["pt_round"][[0, 1, 3]] == -1) and out["rounds"][0]["num_outliers"] == 5


def test_constraint_rows_follow_the_round_and_protection_the_original_index():
    pc = np.zeros((12, 3))
    pc[1] = 7.0
    pc[5] = 9.0
    seen = []
    out = stub_loop([2, 1, 0], seen, min_outliers=0, min_points=1, use_point_constraints=1, points_constraints=pc)
    # round 0 flags original 0 and 3 (1 is protected, 2 has no view); round 1 solves 9 points and is handed rows 0..8 of
    # the caller's array, so row 5 now sits on original point 8 -- while original 5 stays protected and 4 is flagged
    assert out["rounds"][0]["outliers"].tolist() == [0, 3] and out["rounds"][1]["outliers"].tolist() == [4]
    assert [s[0] for s in seen] == [11, 9, 8]
    assert np.array_equal(seen[1][1], pc[:9]) and np.array_equal(seen[2][1], pc[:8])
    assert out["pt_round"][[1, 5]].tolist() == [-1, -1]


def test_inject_outliers_moves_the_chosen_views_only():
    base = synth.crs_scene(synth.ba_scene(6, 80, 3, seed=5))
    for kw, per_point in (({}, 1), ({"all_views": True}, 3), ({"camera": 2}, 1)):
        scene, chosen = synth.inject_outliers(base, 9, seed=4, **kw)
        moved = np.nonzero(np.linalg.norm(scene["projections"] - base["projections"], axis=1) > 0)[0]
        pts_moved = np.repeat(np.arange(80), 3)[moved]
        assert len(chosen) == 9 and np.array_equal(np.unique(pts_moved), chosen) and len(moved) == 9 * per_point
        assert np.linalg.norm(scene["projections"][moved] - base["projections"][moved], axis=1).min() >= 50.0
        if "camera" in kw:
            assert np.all(base["vis_cam"][moved] == 2)
    again, chosen2 = synth.inject_outliers(base, 9, seed=4)
    first, chosen1 = synth.inject_outliers(base, 9, seed=4)
    assert np.array_equal(again["projections"], first["projections"]) and np.array_equal(chosen1, chosen2)


@pytest.mark.parametrize("name", ["stops_small", "protected_quirk", "empty_on_entry", "three_rounds"])
def test_reference_loop_reproduces_the_golden_file(name):
    from oracle import loader
    if loader.ref_sba() is None:
        pytest.skip("oracle/_ref is not built")
    from tests.golden import make_outlier_loop_golden as mk
    scene, kw = scenes.GOLDEN[name]()
    got = mk.flatten(name, mk.reference_loop(scene, kw))
    g = np.load(GOLD)
    for key, val in got.items():
        if key.endswith(("_count", "_sizes", "_pt_round")):
            assert np.array_equal(val, g[key]), key
        else:
            np.testing.assert_allclose(val, g[key], rtol=1e-6, atol=1e-9, err_msg=key)
