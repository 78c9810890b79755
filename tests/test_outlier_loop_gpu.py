"""bsfm_run_sfm_outlier_loop on the GPU (include/bsfm_b200_ba.h).

Composition: the entry against a host loop written here from the single-call entries (bsfm_run_sfm_crs_fe,
bsfm_reprojection_outliers_crs_fe) and the numpy compaction of tests/outlier_loop_restatement.py, bit for bit.
Reference parity: against tests/golden/outlier_loop_golden.npz (the unmodified reference behind the same loop).
Arguments, errors, and the host-to-device bytes of every round."""
import ctypes
import os

import numpy as np
import pytest

from bundler_sfm_b200 import _lib, bundle, synth
from tests import outlier_loop_restatement as rs
from tests import outlier_loop_scenes as scenes

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "outlier_loop_golden.npz")


def host_loop(scene, kw):
    """what a caller had to write before the entry existed"""
    loop_kw, solve_kw, outl_kw = scenes.split_kw(kw)
    fe = solve_kw.pop("optimize_for_fisheye", 0)
    outl_kw.pop("optimize_for_fisheye", None)

    def solve(s, pc):
        return bundle.run_sfm(s, optimize_for_fisheye=fe, points_constraints=pc, **solve_kw)

    def outlier_pass(s, prot):
        return bundle.reprojection_outliers(s, pt_protected=prot, optimize_for_fisheye=fe, **outl_kw)

    return rs.run_loop(scene, solve, outlier_pass, **loop_kw)


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def check_composition(scene, kw, what):
    got = bundle.run_sfm_outlier_loop(scene, **kw)
    want = host_loop(scene, kw)
    assert got["count"] == want["count"], (what, "rounds", got["count"], want["count"])
    for r, (g, w) in enumerate(zip(got["rounds"], want["rounds"])):
        for key in ("num_pts", "nvis", "num_outliers", "removed"):
            assert g[key] == w[key], (what, "round", r, key, g[key], w[key])
        assert same_bytes(g["info"], w["info"]), (what, "round", r, "info", g["info"], w["info"])
        assert same_bytes(g["global_mean"], w["global_mean"]), (what, "round", r, "global_mean")
    assert np.array_equal(got["pt_round"], want["pt_round"]), (what, "pt_round", np.nonzero(got["pt_round"] != want["pt_round"])[0][:10])
    assert same_bytes(got["pt_error"], want["pt_error"]), (what, "pt_error")
    if want["count"]:
        assert same_bytes(got["cam_stats"], want["cam_stats"]), (what, "cam_stats")
    for key in ("R", "c", "f", "k"):
        assert same_bytes(got[key], want[key]), (what, "final cameras", key)
    assert same_bytes(got["pts"], want["pts"]), (what, "final points (init_pts write-back by original index)")
    assert got["mean_error"] == want["mean_error"], (what, "mean_error")
    return got


@pytest.mark.parametrize("name", sorted(scenes.ALL))
def test_composition_on_the_golden_scenes(name):
    scene, kw = scenes.ALL[name]()
    got = check_composition(scene, kw, name)
    if name == "protected_quirk":
        assert got["pt_round"][10] == -1 and got["pt_round"][3] == 0 and got["count"] == 2
    if name == "empty_on_entry":
        assert got["pt_round"][[0, 7, 8, 399]].tolist() == [-2] * 4
        assert same_bytes(got["pts"][[0, 7, 8, 399]], scene["pts"][[0, 7, 8, 399]])
    if name == "too_few":
        assert got["mean_error"] == rs.DBL_MAX


def test_composition_on_a_large_reduced_camera_system():
    """180 cameras x 9 parameters = 1620 unknowns: the large Cholesky path, whose camera order is decided again every round"""
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(180, 6000, 5, seed=91)), 60, seed=92)
    got = check_composition(scene, {"min_outliers": 10}, "180 cameras")
    assert got["count"] >= 2 and got["rounds"][0]["num_outliers"] >= 60


@pytest.mark.parametrize("seed,kw", [
    (101, {"min_outliers": 4}),
    (102, {"min_outliers": 4, "est_focal_length": 1, "undistort": 0}),
    (103, {"remove_outliers": 0}),
])
def test_composition_on_fresh_scenes(seed, kw):
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(12, 900, 4, seed=seed)), 15, seed=seed + 1000, all_views=seed == 102)
    got = check_composition(scene, kw, f"seed {seed}")
    if not kw.get("remove_outliers", 1):     # one solve + one pass, nothing removed
        assert got["count"] == 1 and np.all(got["pt_round"] == -1) and got["rounds"][0]["num_outliers"] >= 15
        one = bundle.run_sfm(scene, optimize_for_fisheye=0)
        assert same_bytes(got["pts"], one["pts"]) and same_bytes(got["R"], one["R"])


def rel_group_err(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("name", sorted(scenes.GOLDEN))
def test_reference_parity(name):
    g = np.load(GOLD)
    scene, kw = scenes.GOLDEN[name]()
    got = bundle.run_sfm_outlier_loop(scene, **kw)
    assert got["count"] == int(g[f"{name}_count"]), (name, "rounds")
    # the same outlier set in every round: the injected errors are gross, no threshold decides membership by rounding
    assert np.array_equal(got["pt_round"], g[f"{name}_pt_round"]), (name, "outlier sets")
    sizes = np.array([[r["num_pts"], r["nvis"], r["num_outliers"]] for r in got["rounds"]]).reshape(-1, 3)
    assert np.array_equal(sizes, g[f"{name}_sizes"]), (name, "sizes")
    info = g[f"{name}_info"]
    equal_iterations = True
    for r, rd in enumerate(got["rounds"]):
        # Snavely's stop-8 rule fires on a statistic that passes its threshold by rounding (tests/test_ba_gpu.py,
        # test_tile_kernel_system_vs_reference), and with gross outliers in the solve it hovers near the threshold for
        # many iterations (the H100 stopped round 0 of protected_quirk after 53 iterations, the reference after 58): the
        # stop reason must agree and the count be within 10 %, at least 3.  The 1e-5 px bounds hold at equal counts; a
        # solve that stopped elsewhere on the same plateau is held to 1e-2 px (protected_quirk keeps a protected
        # gross outlier in the solve: its global mean differs by 1.3e-3 px after 53 against 58 iterations).
        assert int(rd["info"][6]) == int(info[r, 6]), (name, "round", r, "stop reason", rd["info"][6], info[r, 6])
        same = int(rd["info"][5]) == int(info[r, 5])
        # (round 1 of protected_quirk, where the reference itself wanders for 123 iterations, is left to the error bounds)
        if int(info[r, 5]) <= 100:
            assert abs(int(rd["info"][5]) - int(info[r, 5])) <= max(3, int(info[r, 5]) // 10), (name, "round", r, "iterations", rd["info"][5], info[r, 5])
        equal_iterations = equal_iterations and same
        rmse, rmse_ref = np.sqrt(rd["info"][1] / rd["nvis"]), np.sqrt(info[r, 1] / rd["nvis"])
        assert abs(rmse - rmse_ref) <= (1e-5 if same else 1e-2), (name, "round", r, "rmse", rmse, rmse_ref)
        assert abs(rd["global_mean"] - g[f"{name}_global_mean"][r]) <= (1e-5 if same else 1e-2), (name, "round", r, "global mean")
    if name == "too_few":
        assert got["mean_error"] == rs.DBL_MAX == float(g[f"{name}_mean_error"])
    elif equal_iterations:      # a mean of distances of a solution that agrees to 1e-5 px RMSE: the same bound
        assert abs(got["mean_error"] - float(g[f"{name}_mean_error"])) <= 1e-5, (name, "mean_error")
    if equal_iterations:      # after a different number of iterations the weakly determined directions differ
        for key in ("R", "c", "f", "pts"):
            assert rel_group_err(got[key], g[f"{name}_{key}"]) <= 1e-4, (name, key)
        sel = got["pt_round"] >= 0
        assert np.max(np.abs(got["pt_error"][sel] - g[f"{name}_pt_error"][sel]), initial=0.0) <= 1e-4, (name, "pt_error")


def small_scene():
    return synth.inject_outliers(synth.crs_scene(synth.ba_scene(8, 300, 4, seed=111)), 12, seed=112)[0]


def test_faulty_crs_is_refused_with_the_message_of_run_sfm_crs():
    scene = small_scene()
    bad = dict(scene)
    bad["vis_cam"] = scene["vis_cam"].copy()
    bad["vis_cam"][5] = 99
    msgs = []
    for call in (lambda: bundle.run_sfm(bad), lambda: bundle.run_sfm_outlier_loop(bad)):
        with pytest.raises(_lib.BsfmError) as e:
            call()
        msgs.append(str(e.value).split(": ", 1)[-1])
    assert "malformed visibility (CRS) at point 1: camera index outside [0, num_cameras)" in msgs[1]
    assert msgs[0].split("malformed")[-1] == msgs[1].split("malformed")[-1]


def test_rounds_cap_smaller_than_the_rounds_run():
    scene = small_scene()
    full = bundle.run_sfm_outlier_loop(scene, min_outliers=3)
    capped = bundle.run_sfm_outlier_loop(scene, min_outliers=3, rounds_cap=1)
    assert full["count"] >= 2 and capped["count"] == full["count"] and len(capped["rounds"]) == 1
    assert same_bytes(capped["pts"], full["pts"]) and np.array_equal(capped["pt_round"], full["pt_round"])
    none = bundle.run_sfm_outlier_loop(scene, min_outliers=3, rounds_cap=0)
    assert none["count"] == full["count"] and none["rounds"] == []


def test_null_pt_round_and_const_focal_length_are_refused():
    scene = small_scene()
    with pytest.raises(_lib.BsfmError, match="bad arguments"):
        bundle.run_sfm_outlier_loop(scene, pt_round=False)
    lib = bundle.load_library()
    fn = lib.bsfm_run_sfm_outlier_loop
    n, m = len(scene["pts"]), len(scene["R"])
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"])
    pts, rnd, err, mean = scene["pts"].copy(), np.zeros(n, np.int32), np.zeros(n), ctypes.c_double()
    rc = fn(n, m, 0, scene["vis_ptr"].ctypes.data, scene["vis_cam"].ctypes.data, len(scene["vis_cam"]), scene["projections"].ctypes.data,
            1, 1, 1, 1, ctypes.addressof(cams), pts.ctypes.data, 0, 0, None, 0.0, 0, 0, 1e-12, 1, 40, 20, 8.0, 16.0,
            rnd.ctypes.data, err.ctypes.data, None, None, 0, ctypes.byref(mean))
    assert rc < -1, rc
    assert b"const_focal_length" in lib.bsfm_last_error()


def test_rounds_after_the_first_upload_nothing_larger_than_the_camera_tables():
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(10, 4000, 4, seed=121)), 40, seed=122)
    pc = np.zeros((4000, 3))
    pc[17] = scene["gt_pts"][17]
    got = bundle.run_sfm_outlier_loop(scene, min_outliers=5, use_point_constraints=1, points_constraints=pc, point_constraint_weight=1.0)
    assert got["count"] >= 2
    m, nvis0 = 10, len(scene["vis_cam"])
    camera_table = m * ctypes.sizeof(bundle.CameraParams)
    first = got["rounds"][0]
    assert first["h2d_largest"] == nvis0 * 16 and first["h2d_bytes"] >= nvis0 * 20 + 4000 * 28      # the scene goes up once
    for r, rd in enumerate(got["rounds"][1:], 1):
        assert 0 < rd["h2d_largest"] <= camera_table, (r, rd["h2d_largest"], camera_table)
        assert rd["h2d_bytes"] <= 16 * camera_table, (r, rd["h2d_bytes"])
