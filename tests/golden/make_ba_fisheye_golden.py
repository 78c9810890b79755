"""Generates tests/golden/ba_fisheye_golden.npz: run_sfm of the UNMODIFIED reference (oracle/_ref/libref_sba.so, through
loader.run_sfm_ref) with optimize_for_fisheye = 1, i.e. the sfm_project_point2_fisheye projection (lib/sfm-driver/
sfm.c:448-501, selected at :829-856), on scenes made by synth.ba_scene_fisheye:
  ef{0,1}_ud{0,1}  every (est_focal_length, undistort) combination, 10 fisheye cameras / 400 points
  mixed            half of the cameras are ordinary (fisheye = 0) ones
  ki               fisheye and calibrated (known_intrinsics) cameras, alone and together
  cons             RunBundler-style camera constraints (focal prior, distortion weight 100, src/Bundle.cpp:924-974) with
                   ncons = 2 leading cameras fixed, plus point constraints
  fixpts           fix_points = 1 (motion-only sba_mot_levmar with sfm_project_point2_fisheye_mot)
  tcam             explicit_camera_centers = 0 (aj[0..2] = t = -R c)
  export           the V / S / U / W export of the final normal equations (a smaller scene)
  outl             the outlier statistics pass with m_optimize_for_fisheye (src/Bundle.cpp:659-856): the unmodified
                   sfm_project_rd and kth_element_copy around the numpy restatement of ImageData::DistortPoint in
                   tests/fisheye_restatement.py, on the refined ef1_ud1 scene with a nonzero radial distortion, 20 gross
                   measurement errors, one protected point and one fisheye camera with f_focal < 0 (DistortPoint's early
                   return)
Run where the reference sources are, after build():  python tests/golden/make_ba_fisheye_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import loader  # noqa: E402
from bundler_sfm_b200 import synth  # noqa: E402
from tests import fisheye_restatement  # noqa: E402

SCENE_KEYS = ("vmask", "projections", "R", "c", "f", "k", "pts", "fisheye", "fisheye_params")
KI_KEYS = ("known", "K_known", "k_known")
OUT = os.path.join(ROOT, "tests", "golden", "ba_fisheye_golden.npz")


def cases():
    base = synth.ba_scene_fisheye(10, 400, 4, seed=21, ordinary_fraction=0.0)
    out = []
    for ef in (0, 1):
        for ud in (0, 1):
            out.append((f"ef{ef}_ud{ud}", base, {"est_focal_length": ef, "undistort": ud}, {}))
    out.append(("mixed", synth.ba_scene_fisheye(10, 400, 4, seed=22, ordinary_fraction=0.5), {}, {}))
    out.append(("ki", synth.ba_scene_fisheye(10, 400, 4, seed=23, ordinary_fraction=0.3, known_fraction=0.5), {}, {}))
    sc = synth.ba_scene_fisheye(10, 400, 4, seed=24)
    m, n = len(sc["f"]), sc["pts"].shape[0]
    rng = np.random.default_rng(6)
    constrained = np.zeros((m, 9), np.int8); constrained[:, 6:9] = 1
    constraints = np.zeros((m, 9)); constraints[:, 6] = sc["f"]          # focal prior at the initial focal length
    weights = np.zeros((m, 9)); weights[:, 6] = 1e-4; weights[:, 7:9] = 100.0
    pcons = np.zeros((n, 3))
    sel = rng.choice(n, 40, replace=False)
    pcons[sel] = sc["gt_pts"][sel]
    arrays = {"constrained": constrained, "constraints": constraints, "weights": weights, "points_constraints": pcons}
    out.append(("cons", sc, {"ncons": 2, "use_constraints": 1, "use_point_constraints": 1, "point_constraint_weight": 0.05}, arrays))
    out.append(("fixpts", synth.ba_scene_fisheye(10, 400, 4, seed=25), {"fix_points": 1}, {}))
    sc = synth.ba_scene_fisheye(10, 400, 4, seed=26)
    R = sc["R"].reshape(-1, 3, 3)
    sc = dict(sc, c=-np.einsum("jab,jb->ja", R, sc["c"]))      # translations for explicit_camera_centers = 0
    out.append(("tcam", sc, {"explicit_camera_centers": 0}, {}))
    out.append(("export", synth.ba_scene_fisheye(6, 150, 3, seed=27), {"export": True}, {}))
    return out


def outlier_case(scene, ref):
    """refined scene with a radial distortion, 20 gross errors, one protected point, one camera with f_focal < 0"""
    rng = np.random.default_rng(9)
    m = len(ref["f"])
    params = scene["fisheye_params"].copy()
    params[1, 4] = -params[1, 4]
    sc = dict(scene, R=ref["R"], c=ref["c"], f=ref["f"], k=rng.uniform(-0.03, 0.03, (m, 2)), pts=ref["pts"], fisheye_params=params)
    proj = sc["projections"].copy()
    bad = rng.choice(len(proj), 20, replace=False)
    proj[bad] += rng.normal(0, 40.0, (20, 2))
    sc["projections"] = proj
    prot = np.zeros(sc["pts"].shape[0], np.int8)
    pi = np.nonzero(sc["vmask"])[0]
    prot[pi[bad[0]]] = 1
    return sc, prot, fisheye_restatement.reprojection_outliers_fisheye(sc, 1, 2.0, 16.0, prot)


def main():
    assert loader.ref_sba() is not None, "build oracle/_ref first"
    out = {}
    solved = {}
    for name, scene, kw, arrays in cases():
        for k in SCENE_KEYS + KI_KEYS:
            if k in scene:
                out[f"{name}_{k}"] = scene[k]
        for k, v in kw.items():
            out[f"{name}_kw_{k}"] = np.array(v)
        for k, v in arrays.items():
            out[f"{name}_{k}"] = v
        ref = loader.run_sfm_ref(scene, optimize_for_fisheye=1, **kw, **arrays, **synth.fe_kwargs(scene))
        for k in ("R", "c", "f", "k", "pts", "info") + (("V", "S", "U", "W") if kw.get("export") else ()):
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
