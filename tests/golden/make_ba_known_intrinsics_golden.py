"""Generates tests/golden/ba_known_intrinsics_golden.npz: run_sfm of the UNMODIFIED reference (oracle/_ref/libref_sba.so,
through loader.run_sfm_ref) on scenes of calibrated cameras (camera_params_t::known_intrinsics, K_known, k_known;
lib/sfm-driver/sfm.c:339-357), made by synth.ba_scene_known_intrinsics:
  ef{0,1}_ud{0,1}  every (est_focal_length, undistort) combination, 10 calibrated cameras / 400 points
  mixed            half of the cameras are ordinary focal-only cameras
  cons             camera constraints (ncons = 2 leading cameras fixed, weighted centres) plus point constraints
  fixpts           fix_points = 1 (motion-only sba_mot_levmar)
  tcam             explicit_camera_centers = 0 (aj[0..2] = t = -R c)
  outl             the outlier statistics pass (src/Bundle.cpp:659-856) on the refined ef1_ud1 scene with 20 gross
                   measurement errors and one protected point, computed like the reference leg of
                   oracle/outlier_oracle.py: the unmodified sfm_project_rd (which reads the calibration from the camera
                   struct) and kth_element_copy, driven by the same loop
Run where the reference sources are, after build():  python tests/golden/make_ba_known_intrinsics_golden.py"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import loader, outlier_oracle  # noqa: E402
from bundler_sfm_b200 import bundle, synth  # noqa: E402

SCENE_KEYS = ("vmask", "projections", "R", "c", "f", "k", "pts", "known", "K_known", "k_known")
OUT = os.path.join(ROOT, "tests", "golden", "ba_known_intrinsics_golden.npz")


def cases():
    base = synth.ba_scene_known_intrinsics(10, 400, 4, seed=11)
    out = []
    for ef in (0, 1):
        for ud in (0, 1):
            out.append((f"ef{ef}_ud{ud}", base, {"est_focal_length": ef, "undistort": ud}, {}))
    out.append(("mixed", synth.ba_scene_known_intrinsics(10, 400, 4, seed=12, ordinary_fraction=0.5), {}, {}))
    sc = synth.ba_scene_known_intrinsics(10, 400, 4, seed=13)
    m, n = len(sc["f"]), sc["pts"].shape[0]
    rng = np.random.default_rng(5)
    constrained = np.zeros((m, 9), np.int8); constrained[:, 0:3] = 1
    constraints = np.zeros((m, 9)); constraints[:, 0:3] = sc["gt_c"]
    weights = np.zeros((m, 9)); weights[:, 0:3] = 1e3
    pcons = np.zeros((n, 3))
    sel = rng.choice(n, 40, replace=False)
    pcons[sel] = sc["gt_pts"][sel]
    arrays = {"constrained": constrained, "constraints": constraints, "weights": weights, "points_constraints": pcons}
    out.append(("cons", sc, {"ncons": 2, "use_constraints": 1, "use_point_constraints": 1, "point_constraint_weight": 0.05}, arrays))
    out.append(("fixpts", synth.ba_scene_known_intrinsics(10, 400, 4, seed=14), {"fix_points": 1}, {}))
    sc = synth.ba_scene_known_intrinsics(10, 400, 4, seed=15)
    R = sc["R"].reshape(-1, 3, 3)
    sc = dict(sc, c=-np.einsum("jab,jb->ja", R, sc["c"]))      # translations for explicit_camera_centers = 0
    out.append(("tcam", sc, {"explicit_camera_centers": 0}, {}))
    return out


def reference_outliers(sc, min_thresh, max_thresh, prot):
    """the loop of outlier_oracle.reprojection_outliers with its reference building blocks, on camera structs that carry
    the calibration (known_intrinsics, K_known, k_known)"""
    lib = loader.ref_sba()
    fn = lib.sfm_project_rd
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int, ctypes.c_int]
    kth = lib.kth_element_copy
    kth.restype = ctypes.c_double
    kth.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    cams = bundle.make_cameras(sc["R"], sc["c"], sc["f"], sc["k"], known=sc["known"], K_known=sc["K_known"], k_known=sc["k_known"])
    pts = np.ascontiguousarray(sc["pts"], dtype=np.float64)
    obs_pt, obs_cam = np.nonzero(np.asarray(sc["vmask"]) != 0)
    size = ctypes.sizeof(bundle.CameraParams)
    base = ctypes.addressof(cams)
    dist = np.zeros(len(obs_pt))
    for o, (i, j) in enumerate(zip(obs_pt, obs_cam)):
        cam = bundle.CameraParams.from_address(base + int(j) * size)
        K = (ctypes.c_double * 9)(cam.f, 0, 0, 0, cam.f, 0, 0, 0, 1)                        # Bundle.cpp:670-672
        dt = (ctypes.c_double * 3)(cam.t[0], cam.t[1], cam.t[2])
        b = (ctypes.c_double * 3)(*pts[i])
        pr = (ctypes.c_double * 2)()
        fn(base + int(j) * size, K, ctypes.addressof(cam) + bundle.CameraParams.k.offset, ctypes.addressof(cam), dt, b, pr, 1, 1)
        dx, dy = pr[0] - sc["projections"][o, 0], pr[1] - sc["projections"][o, 1]
        dist[o] = np.sqrt(dx * dx + dy * dy)                                                 # Bundle.cpp:750-753
    m = len(sc["f"])
    stats = np.zeros((m, 5))
    outliers, errors, first_cam = [], [], []
    tot, cnt = 0.0, 0
    for j in range(m):
        sel = np.nonzero(obs_cam == j)[0]
        d = np.ascontiguousarray(dist[sel])
        nj = len(d)
        k80, k50 = outlier_oracle.iround(0.8 * nj), outlier_oracle.iround(0.5 * nj)
        med80 = kth(nj, k80, d.ctypes.data) if k80 < nj else 0.0
        med50 = kth(nj, k50, d.ctypes.data) if k50 < nj else 0.0
        thresh = 1.2 * 2.0 * med80
        thresh = min_thresh if thresh < min_thresh else (max_thresh if thresh > max_thresh else thresh)
        s = 0.0
        for v in d:
            s += v
        stats[j] = (nj, s / nj if nj else np.nan, med50, med80, thresh)
        tot += s; cnt += nj
        for q, o in enumerate(sel):
            i = int(obs_pt[o])
            if prot[i]:
                continue
            if d[q] > thresh and i not in outliers:
                outliers.append(i); errors.append(float(d[q])); first_cam.append(j)
    order = sorted(range(len(outliers)), key=lambda q: (first_cam[q], outliers[q]))
    return {"dist": dist, "stats": stats, "outliers": np.array([outliers[q] for q in order], dtype=np.int32),
            "errors": np.array([errors[q] for q in order]), "global_mean": tot / cnt}


def outlier_case(scene, ref):
    """refined scene + 20 gross errors + one protected point"""
    rng = np.random.default_rng(8)
    sc = dict(scene, R=ref["R"], c=ref["c"], f=ref["f"], k=ref["k"], pts=ref["pts"])
    proj = sc["projections"].copy()
    bad = rng.choice(len(proj), 20, replace=False)
    proj[bad] += rng.normal(0, 40.0, (20, 2))
    sc["projections"] = proj
    prot = np.zeros(sc["pts"].shape[0], np.int8)
    pi = np.nonzero(sc["vmask"])[0]
    prot[pi[bad[0]]] = 1
    return sc, prot, reference_outliers(sc, 2.0, 16.0, prot)


def main():
    assert loader.ref_sba() is not None, "build oracle/_ref first"
    out = {}
    solved = {}
    for name, scene, kw, arrays in cases():
        for k in SCENE_KEYS:
            out[f"{name}_{k}"] = scene[k]
        for k, v in kw.items():
            out[f"{name}_kw_{k}"] = np.array(v)
        for k, v in arrays.items():
            out[f"{name}_{k}"] = v
        ref = loader.run_sfm_ref(scene, **kw, **arrays, **synth.ki_kwargs(scene))
        for k in ("R", "c", "f", "k", "pts", "info"):
            out[f"{name}_ref_{k}"] = ref[k]
        solved[name] = (scene, ref)
        nvis = scene["projections"].shape[0]
        print(f"{name:8s} it {int(ref['info'][5]):3d} stop {int(ref['info'][6])} rmse {np.sqrt(ref['info'][0] / nvis):.4f} -> "
              f"{np.sqrt(ref['info'][1] / nvis):.6f}")
    sc, prot, r = outlier_case(*solved["ef1_ud1"])
    for k in SCENE_KEYS:
        out[f"outl_{k}"] = sc[k]
    out["outl_protected"] = prot
    out["outl_thresholds"] = np.array([2.0, 16.0])
    for k in ("dist", "stats", "outliers", "errors"):
        out[f"outl_ref_{k}"] = r[k]
    out["outl_ref_global_mean"] = np.array(r["global_mean"])
    print("outl     observations", len(r["dist"]), "outliers", len(r["outliers"]), "global mean", r["global_mean"])
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
