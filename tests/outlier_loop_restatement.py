"""numpy restatement of the do / while of BundlerApp::RunSFM_SBA (src/Bundle.cpp:588-913), the loop that
bsfm_run_sfm_outlier_loop runs on the GPU.  The solve and the outlier pass are callables, so the same loop runs over
the unmodified reference (tests/golden/make_outlier_loop_golden.py), over the library's single-call entries (the
composition test) or over stubs."""
import numpy as np

DBL_MAX = np.finfo(np.float64).max
CAMERA_KEYS = ("R", "c", "f", "k")


def compact_crs(vis_ptr, vis_cam, projections, keep):
    """the points with keep[i] set, renumbered densely in ascending order (remap, Bundle.cpp:614-636), with their views
    -> (vis_ptr, vis_cam, projections, orig), orig[q] = the old index of new point q"""
    vis_ptr = np.asarray(vis_ptr, dtype=np.int64)
    keep = np.asarray(keep, dtype=bool)
    views = np.diff(vis_ptr)
    orig = np.nonzero(keep)[0]
    obs_keep = np.repeat(keep, views)
    new_ptr = np.concatenate([[0], np.cumsum(views[orig])]).astype(np.int32)
    return new_ptr, np.asarray(vis_cam)[obs_keep].astype(np.int32), np.asarray(projections, dtype=np.float64).reshape(-1, 2)[obs_keep], orig


def run_loop(scene, solve, outlier_pass, remove_outliers=1, min_outliers=40, min_points=20,
             use_point_constraints=0, points_constraints=None):
    """scene: a CRS scene dict (synth.crs_scene).
    solve(round_scene, points_constraints) -> dict with R, c, f, k, pts, info: run_sfm on the round's compacted scene.
        QUIRK: points_constraints is the FIRST len(round points) rows of the caller's array, not the rows of the round's
        points: the reference passes m_point_constraints to run_sfm as it is (Bundle.cpp:651, sfm.c:757-781).
    outlier_pass(round_scene, pt_protected) -> dict with stats, outliers, errors, global_mean, on the solved round scene;
        pt_protected follows the ORIGINAL index (Bundle.cpp:800-806).
    Returns count, R, c, f, k, pts, pt_round, pt_error, cam_stats, rounds, mean_error like bundle.run_sfm_outlier_loop;
    every round also lists its `outliers` by original index."""
    n = len(scene["pts"])
    vis_ptr = np.asarray(scene["vis_ptr"], dtype=np.int64)
    alive = np.diff(vis_ptr) > 0
    pt_round = np.where(alive, -1, -2).astype(np.int32)
    pt_error = np.zeros(n)
    pts = np.array(scene["pts"], dtype=np.float64)
    cams = {k: np.array(scene[k], dtype=np.float64) for k in CAMERA_KEYS}
    pc = None if not use_point_constraints else np.asarray(points_constraints, dtype=np.float64)
    rounds, total_outliers, mean_error, cam_stats = [], 0, 0.0, None
    while True:
        if n - total_outliers < min_points:                                  # :588-595, on the original num_pts
            mean_error = DBL_MAX
            break
        ptr, cam, proj, orig = compact_crs(vis_ptr, scene["vis_cam"], scene["projections"], alive)
        rs = dict(scene)
        rs.update(cams)
        rs.update(vis_ptr=ptr, vis_cam=cam, projections=proj, pts=pts[orig])
        rs.pop("nvis", None)
        sol = solve(rs, None if pc is None else pc[:len(orig)])              # the quirk
        for k in CAMERA_KEYS:
            cams[k] = np.array(sol[k], dtype=np.float64)
        rs.update(cams)
        rs["pts"] = np.array(sol["pts"], dtype=np.float64)
        prot = None if pc is None else (pc[orig, 0] != 0.0).astype(np.int8)  # :800-806
        op = outlier_pass(rs, prot)
        pts[orig] = rs["pts"]                                                # :905-909
        out = np.asarray(op["outliers"], dtype=np.int64)
        rounds.append({"num_pts": len(orig), "nvis": len(cam), "num_outliers": len(out), "removed": int(bool(remove_outliers)),
                       "info": np.array(sol["info"], dtype=np.float64), "global_mean": float(op["global_mean"]),
                       "outliers": np.sort(orig[out])})
        mean_error, cam_stats = float(op["global_mean"]), np.array(op["stats"])
        if not remove_outliers:                                              # :858, :911
            break
        pt_round[orig[out]] = len(rounds) - 1                                # :871-889
        pt_error[orig[out]] = np.asarray(op["errors"], dtype=np.float64)
        alive[orig[out]] = False
        total_outliers += len(out)
        if not len(out) > min_outliers:                                      # :913
            break
    return {"count": len(rounds), **cams, "pts": pts, "pt_round": pt_round, "pt_error": pt_error, "cam_stats": cam_stats,
            "rounds": rounds, "mean_error": mean_error}


def dense_scene(scene):
    """a CRS scene with the dense vmask the reference takes"""
    from bundler_sfm_b200 import bundle
    pi, cj = bundle.observations(scene)
    vmask = np.zeros((len(scene["pts"]), len(scene["R"])), np.int8)
    vmask[pi, cj] = 1
    out = {k: v for k, v in scene.items() if k not in ("vis_ptr", "vis_cam", "nvis")}
    out["vmask"] = vmask
    return out
