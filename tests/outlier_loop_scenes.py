"""The scenes of the outlier-loop tests, rebuilt from seeds: name -> (CRS scene, keywords of bundle.run_sfm_outlier_loop).
tests/golden/make_outlier_loop_golden.py runs the reference over them; the GPU tests run the library."""
import os

import numpy as np

from bundler_sfm_b200 import synth

BA_GOLD = os.path.join(os.path.dirname(__file__), "golden", "ba_golden.npz")
LOOP_KEYS = ("remove_outliers", "min_outliers", "min_points", "use_point_constraints", "points_constraints")
CAMERA_KW = ("known", "K_known", "k_known", "fisheye", "fisheye_params")


def kermit():
    g = np.load(BA_GOLD)
    scene = synth.crs_scene({k: g[f"kermit_{k}"] for k in ("vmask", "projections", "R", "c", "f", "k", "pts")})
    scene, _ = synth.inject_outliers(scene, 12, seed=11)
    return scene, {}


def three_rounds():
    """camera 0 has 30 % of its views displaced by >= 60 px, so its threshold is the upper clamp (16 px) in round 0 and
    the 12-14 px displacements of 15 more of its views pass; round 1 lowers it to 8 px and flags those; round 2 flags
    nothing"""
    scene = synth.crs_scene(synth.ba_scene(8, 600, 4, seed=21))
    scene, gross = synth.inject_outliers(scene, 90, seed=22, displacement=60.0, camera=0)
    from bundler_sfm_b200 import bundle
    pi, cj = bundle.observations(scene)
    rest = np.setdiff1d(pi[cj == 0], gross)
    rng = np.random.default_rng(23)
    mild = np.sort(rng.choice(rest, size=15, replace=False))
    proj = scene["projections"].copy()
    for i in mild:
        o = np.nonzero((pi == i) & (cj == 0))[0][0]
        ang = rng.uniform(0.0, 2.0 * np.pi)
        proj[o] += rng.uniform(12.0, 14.0) * np.array([np.cos(ang), np.sin(ang)])
    scene["projections"] = proj
    return scene, {"min_outliers": 5}


def stops_small():
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(10, 500, 4, seed=31)), 7, seed=32)
    return scene, {"est_focal_length": 0, "undistort": 0}


def too_few():
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(9, 300, 5, seed=41)), 30, seed=42)
    return scene, {"min_outliers": 5, "min_points": 280}


def protected_quirk():
    """point 10 is constrained, hence protected, and a gross outlier; point 3, below it, is removed in round 0, so in
    round 1 the solver's constraint of row 10 acts on original point 11 while original point 10 stays protected"""
    base = synth.ba_scene(8, 400, 4, seed=51)
    scene, chosen = synth.inject_outliers(synth.crs_scene(base), 6, seed=52, candidates=[3, 10, 50, 51, 120, 300])
    assert 3 in chosen and 10 in chosen, chosen
    pc = np.zeros((400, 3))
    for i in (10, 200):
        pc[i] = base["gt_pts"][i]
    return scene, {"min_outliers": 2, "use_point_constraints": 1, "points_constraints": pc, "point_constraint_weight": 100.0}


def empty_on_entry():
    base = synth.ba_scene(8, 400, 4, seed=61)
    base["vmask"][[0, 7, 8, 399], :] = 0
    keep = np.ones(400, bool); keep[[0, 7, 8, 399]] = False
    base["projections"] = base["projections"][np.repeat(keep, 4)]
    scene, _ = synth.inject_outliers(synth.crs_scene(base), 8, seed=62)
    return scene, {"min_outliers": 3}


def fix_points():
    scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(8, 400, 4, seed=71, pt_noise=0.002)), 8, seed=72)
    return scene, {"min_outliers": 3, "fix_points": 1}


def fisheye():
    base = synth.ba_scene_fisheye(10, 400, 4, seed=81)
    scene, _ = synth.inject_outliers(synth.crs_scene(base), 8, seed=82)
    return scene, {"min_outliers": 3, "optimize_for_fisheye": 1, **synth.fe_kwargs(base)}


# the scenes the reference has run (tests/golden/outlier_loop_golden.npz), and the fisheye scene, whose DistortPoint step
# the CPU oracle of the outlier pass does not have: the library's own entries cover it (composition)
GOLDEN = {f.__name__: f for f in (kermit, three_rounds, stops_small, too_few, protected_quirk, empty_on_entry, fix_points)}
ALL = dict(GOLDEN, fisheye=fisheye)


def split_kw(kw):
    """keywords of bundle.run_sfm_outlier_loop -> (those of the loop restatement, of run_sfm, of reprojection_outliers)"""
    loop = {k: kw[k] for k in LOOP_KEYS if k in kw}
    cams = {k: kw[k] for k in CAMERA_KW if k in kw}
    solve = {k: kw[k] for k in ("est_focal_length", "undistort", "fix_points", "use_point_constraints", "point_constraint_weight",
                                "optimize_for_fisheye", "ncons", "eps2") if k in kw}
    outl = {"estimate_distortion": kw.get("undistort", 1), "min_thresh": kw.get("min_thresh", 8.0), "max_thresh": kw.get("max_thresh", 16.0)}
    if "optimize_for_fisheye" in kw:
        outl["optimize_for_fisheye"] = kw["optimize_for_fisheye"]
    return loop, dict(solve, **cams), dict(outl, **cams)
