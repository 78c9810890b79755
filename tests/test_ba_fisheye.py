"""Bundle adjustment and the outlier pass of fisheye cameras (run_sfm's optimize_for_fisheye, what
`bundler --optimize_for_fisheye` sets up; camera_params_t::fisheye, f_cx, f_cy, f_rad, f_angle, f_focal).

CPU tests pin the committed outputs of the unmodified reference (tests/golden/ba_fisheye_golden.npz, made by
tests/golden/make_ba_fisheye_golden.py) with the numpy restatements of tests/fisheye_restatement.py, and the host
sfm_project_point2_fisheye of the run_sfm shim against numpy.  GPU tests run every golden case through bsfm_run_sfm_fe and
the other _fe entries.

Tolerances as in tests/test_ba_known_intrinsics.py: final reprojection RMSE within 1e-5 px, same iteration count and
stop reason (motion-only: a rounding-driven stop), parameters within 1e-4 of each group's largest magnitude, initial
error within 1e-9 relative.  The device atan and the C library's differ in the last bits, so no result is bitwise
the reference's."""
import ctypes
import math
import os

import numpy as np
import pytest

from bundler_sfm_b200 import bundle, synth
from bundler_sfm_b200._lib import BsfmError, last_error
from tests import fisheye_restatement as FR
from tests.test_ba_known_intrinsics import project_ref, rot_update

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ba_fisheye_golden.npz")
SHIM = os.path.join(ROOT, "shim", "_build")
SCENE_KEYS = ("vmask", "projections", "R", "c", "f", "k", "pts", "fisheye", "fisheye_params", "known", "K_known", "k_known")
MOTSTR_CASES = ("ef0_ud0", "ef0_ud1", "ef1_ud0", "ef1_ud1", "mixed", "ki", "cons", "tcam", "export")
SOLVE_CASES = MOTSTR_CASES + ("fixpts",)
RMSE_TOL = 1e-5
PARAM_TOL = 1e-4


def gold():
    return np.load(GOLD)


def gold_case(g, name):
    scene = {k: g[f"{name}_{k}"] for k in SCENE_KEYS if f"{name}_{k}" in g.files}
    kw = {k[len(name) + 4:]: g[k].item() for k in g.files if k.startswith(f"{name}_kw_")}
    for k in ("constrained", "constraints", "weights", "points_constraints"):
        if f"{name}_{k}" in g.files:
            kw[k] = g[f"{name}_{k}"]
    ref = {k: g[f"{name}_ref_{k}"] for k in ("R", "c", "f", "k", "pts", "info", "V", "S", "U", "W") if f"{name}_ref_{k}" in g.files}
    return scene, kw, ref


def rel_group_err(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def check_solution(got, ref, nvis, what, fixed_pts=None):
    r_gpu, r_ref = np.sqrt(got["info"][1] / nvis), np.sqrt(ref["info"][1] / nvis)
    assert abs(r_gpu - r_ref) <= RMSE_TOL, (what, r_gpu, r_ref)
    if fixed_pts is None:
        assert int(got["info"][5]) == int(ref["info"][5]), (what, "iterations", got["info"][5], ref["info"][5])
        assert int(got["info"][6]) == int(ref["info"][6]), (what, "stop reason", got["info"][6], ref["info"][6])
    else:
        # motion-only solves stop through rule 4 with eps4 = 0, i.e. when it holds by ROUNDING at convergence
        # (sba_levmar.c:2596), or through rule 2 (see tests/test_ba_known_intrinsics.py)
        assert int(got["info"][6]) in (2, 4), (what, "stop reason", got["info"][6])
    for key in ("R", "c", "pts", "f"):
        err = rel_group_err(got[key], ref[key])
        assert err <= PARAM_TOL, (what, key, err)
    # the k columns of the fisheye Jacobian are zero: only camera constraints move k
    assert np.max(np.abs(got["k"] - ref["k"])) * 5.0 <= PARAM_TOL * max(1.0, 5.0 * np.max(np.abs(ref["k"]))), (what, "k")
    assert abs(got["info"][0] - ref["info"][0]) <= 1e-9 * abs(ref["info"][0]), (what, "initial error")
    if fixed_pts is not None:
        assert np.array_equal(got["pts"], fixed_pts), (what, "points must stay fixed")


def fe(scene):
    return synth.fe_kwargs(scene)


def golden_kw(kw):
    return {k: v for k, v in kw.items() if k != "export"}


# ---- CPU: the golden file against the numpy restatements ------------------------------------------------------------
def test_golden_scenes_cover_the_cases():
    g = gold()
    scene, _, _ = gold_case(g, "mixed")
    assert sorted(set(scene["fisheye"].tolist())) == [0, 1]
    scene, _, _ = gold_case(g, "ki")
    assert ((scene["known"] != 0) & (scene["fisheye"] != 0)).any() and ((scene["known"] != 0) & (scene["fisheye"] == 0)).any()
    assert (gold_case(g, "cons")[1]["weights"][:, 7:9] == 100.0).all()
    assert (g["outl_fisheye_params"][:, 4] < 0).sum() == 1


@pytest.mark.parametrize("name", MOTSTR_CASES)
def test_cpu_restatement_reproduces_golden(name):
    """the numpy restatement of run_sfm with sfm_project_point2_fisheye reproduces the unmodified reference's outputs"""
    g = gold()
    scene, kw, ref = gold_case(g, name)
    ki = {k: scene[k] for k in ("known", "K_known", "k_known") if k in scene}
    got = FR.port_run_sfm_fisheye(scene, scene["fisheye"], scene["fisheye_params"], **golden_kw(kw), **ki)
    assert got is not None
    check_solution(got, ref, scene["projections"].shape[0], "port_" + name)


def test_cpu_outlier_restatement_reproduces_golden():
    """the outlier pass restated on numpy's projection port (no reference library needed) gives the golden case"""
    g = gold()
    sc = {k: g[f"outl_{k}"] for k in SCENE_KEYS if f"outl_{k}" in g.files}
    lo, hi = g["outl_thresholds"]
    r = FR.reprojection_outliers_fisheye(sc, 1, float(lo), float(hi), g["outl_protected"], use_reference=False)
    assert np.allclose(r["dist"], g["outl_ref_dist"], rtol=1e-12, atol=1e-12)
    assert np.array_equal(r["stats"][:, 0], g["outl_ref_stats"][:, 0])
    assert np.allclose(r["stats"][:, 1:], g["outl_ref_stats"][:, 1:], rtol=1e-12, atol=1e-12)
    assert np.array_equal(r["outliers"], g["outl_ref_outliers"])
    assert np.allclose(r["errors"], g["outl_ref_errors"], rtol=1e-12)
    # the camera with f_focal < 0 keeps its undistorted projections (DistortPoint's early return)
    j = int(np.nonzero(sc["fisheye_params"][:, 4] < 0)[0][0])
    plain = FR.reprojection_outliers_fisheye(sc, 1, float(lo), float(hi), g["outl_protected"], optimize_for_fisheye=0,
                                             use_reference=False)
    cam = np.nonzero(sc["vmask"])[1]
    assert np.array_equal(r["dist"][cam == j], plain["dist"][cam == j])
    assert not np.allclose(r["dist"][cam != j], plain["dist"][cam != j])


def test_rotation_of_distort_point_is_the_identity_up_to_rounding():
    R = np.array(FR.R_DISTORT).reshape(3, 3)
    assert np.allclose(R, np.diag([1.0, 1.0, -1.0]), atol=1e-16) and not np.array_equal(R, np.diag([1.0, 1.0, -1.0]))


# ---- CPU: the host sfm_project_point2_fisheye of libsfmdrv_b200.so --------------------------------------------------
class SfmGlobal(ctypes.Structure):
    """== bsfm_sfm_global_t / sfm_global_t (lib/sfm-driver/sfm.c:39-54)"""
    _fields_ = [("num_cameras", ctypes.c_int), ("num_points", ctypes.c_int), ("num_params_per_camera", ctypes.c_int),
                ("est_focal_length", ctypes.c_int), ("const_focal_length", ctypes.c_int),
                ("explicit_camera_centers", ctypes.c_int), ("estimate_distortion", ctypes.c_int),
                ("global_params", bundle.CameraParams), ("init_params", ctypes.c_void_p), ("points", ctypes.c_void_p)]


def _sfmdrv():
    path = os.path.join(SHIM, "libsfmdrv_b200.so")
    if not os.path.exists(path):
        pytest.skip("shim/_build not built")
    bundle.load_library()
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
    for name in ("sfm_project_point2_fisheye", "sfm_project_point3"):
        getattr(lib, name).argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        getattr(lib, name).restype = None
    lib.sfm_project_point2_fisheye_mot.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.sfm_project_point2_fisheye_mot.restype = None
    return lib


def _globals(sc, cams, est_focal, undistort, explicit_centers):
    g = SfmGlobal()
    g.num_cameras, g.num_points = len(sc["f"]), sc["pts"].shape[0]
    g.num_params_per_camera = 6 + est_focal + 2 * undistort
    g.est_focal_length, g.explicit_camera_centers, g.estimate_distortion = est_focal, explicit_centers, undistort
    g.init_params = ctypes.addressof(cams)
    return g


@pytest.mark.parametrize("est_focal,undistort", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("explicit_centers", [1, 0])
def test_shim_host_fisheye_projection_matches_numpy(est_focal, undistort, explicit_centers):
    lib = _sfmdrv()
    sc = synth.ba_scene_fisheye(8, 50, 3, seed=3, ordinary_fraction=0.25, known_fraction=0.25)
    m = len(sc["f"])
    rng = np.random.default_rng(est_focal * 2 + undistort)
    k_rad = rng.uniform(-0.05, 0.05, (m, 2))
    cams = bundle.make_cameras(sc["R"], sc["c"], sc["f"], k_rad, **fe(sc))
    for j in range(m):
        cams[j].f_scale, cams[j].k_scale = 0.001, 5.0
    g = _globals(sc, cams, est_focal, undistort, explicit_centers)
    pts = np.ascontiguousarray(sc["pts"], np.float64)
    g.points = pts.ctypes.data
    worst = 0.0
    for j in range(m):
        for i in range(0, sc["pts"].shape[0], 7):
            w = rng.normal(0, 0.02, 3)
            dt = sc["c"][j] if explicit_centers else -np.asarray(sc["R"][j]).reshape(3, 3) @ sc["c"][j]
            a = list(dt) + list(w)
            if est_focal:
                a.append(sc["f"][j] * 1.01 * 0.001)
            if undistort:
                a += list(k_rad[j] * 5.0)
            a = np.array(a)
            out, out_mot = np.zeros(2), np.zeros(2)
            lib.sfm_project_point2_fisheye(j, i, a.ctypes.data, pts[i].ctypes.data, out.ctypes.data, ctypes.addressof(g))
            lib.sfm_project_point2_fisheye_mot(j, i, a.ctypes.data, out_mot.ctypes.data, ctypes.addressof(g))
            assert np.array_equal(out, out_mot)
            # numpy: the pinhole of sfm_project2 (sfm_project_rd without the radial step), then the mapping
            f = a[6] / 0.001 if est_focal else sc["f"][j]
            kn = "known" in sc and sc["known"][j]
            pin = np.array(project_ref(rot_update(sc["R"][j], w), dt, pts[i], f, None, 0, explicit_centers, kn,
                                       sc["K_known"][j] if kn else None, sc["k_known"][j] if kn else None))
            want = synth.fisheye_map(pin[None], sc["fisheye_params"][j][None])[0] if sc["fisheye"][j] else pin
            worst = max(worst, float(np.max(np.abs(out - want) / np.maximum(np.abs(want), 1.0))))
    assert worst <= 1e-12, worst


def test_shim_host_fisheye_projection_is_nan_on_the_principal_axis():
    """r = 0 is 0/0 in sfm_fisheye_distort: NaN, as in the reference (which does not guard it)"""
    lib = _sfmdrv()
    R = np.eye(3).reshape(1, 9)
    cams = bundle.make_cameras(R, [[0.0, 0.0, 0.0]], [700.0], [[0.0, 0.0]], fisheye=[1],
                               fisheye_params=[[3.0, -2.0, 1000.0, 180.0, 650.0]])
    sc = {"f": [700.0], "pts": np.zeros((1, 3))}
    g = _globals(sc, cams, 0, 0, 1)
    a = np.zeros(6)
    b = np.array([0.0, 0.0, -5.0])
    out = np.zeros(2)
    lib.sfm_project_point2_fisheye(0, 0, a.ctypes.data, b.ctypes.data, out.ctypes.data, ctypes.addressof(g))
    assert np.isnan(out).all()
    b = np.array([0.3, -0.2, -5.0])
    lib.sfm_project_point2_fisheye(0, 0, a.ctypes.data, b.ctypes.data, out.ctypes.data, ctypes.addressof(g))
    u = np.array([-0.3 * 700.0 / -5.0, 0.2 * 700.0 / -5.0])
    r = math.hypot(*u)
    rnew = 1000.0 * (180.0 * math.atan(r / 650.0) / math.pi) / 90.0
    assert np.allclose(out, u * (rnew / r) + np.array([3.0, -2.0]), rtol=1e-14, atol=0)


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", SOLVE_CASES)
def test_golden_cases_through_run_sfm_fe(name):
    g = gold()
    scene, kw, ref = gold_case(g, name)
    got = bundle.run_sfm(scene, optimize_for_fisheye=1, **kw, **fe(scene))
    check_solution(got, ref, scene["projections"].shape[0], name, fixed_pts=scene["pts"] if kw.get("fix_points") else None)
    if kw.get("export"):
        for key in ("V", "S", "U", "W"):
            assert rel_group_err(got[key], ref[key]) <= 1e-3, (key, rel_group_err(got[key], ref[key]))
    crs = bundle.run_sfm(synth.crs_scene(scene), optimize_for_fisheye=1, **kw, **fe(scene))
    for key in ("R", "c", "f", "k", "pts", "info") + (("V", "S", "U", "W") if kw.get("export") else ()):
        assert np.array_equal(crs[key], got[key]), (name, "crs", key)


def _ref_or_skip():
    from oracle import loader
    if loader.ref_sba() is None:
        pytest.skip("oracle/_ref/libref_sba.so not available (the C restatement oracle/ba_oracle.c has no fisheye branch)")
    return loader


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,kw", [
    (20, 2000, {}),
    (16, 1500, {"est_focal_length": 0, "undistort": 1}),
    (180, 4000, {}),     # cnp = 9: reduced system 1620 > 1536 unknowns -> the large Cholesky path
])
def test_fresh_scene_vs_reference(m, n, kw):
    loader = _ref_or_skip()
    scene = synth.ba_scene_fisheye(m, n, 5, seed=m + 3, ordinary_fraction=0.25, known_fraction=0.2)
    got = bundle.run_sfm(scene, optimize_for_fisheye=1, **kw, **fe(scene))
    ref = loader.run_sfm_ref(scene, optimize_for_fisheye=1, **kw, **fe(scene))
    check_solution(got, ref, scene["projections"].shape[0], f"fresh{m}")
    assert got["info"][1] < 0.1 * got["info"][0]


@pytest.mark.gpu
def test_motion_only_fresh_scene_vs_reference():
    loader = _ref_or_skip()
    scene = synth.ba_scene_fisheye(30, 3000, 5, seed=43, ordinary_fraction=0.3)
    got = bundle.run_sfm(scene, optimize_for_fisheye=1, fix_points=1, **fe(scene))
    ref = loader.run_sfm_ref(scene, optimize_for_fisheye=1, fix_points=1, **fe(scene))
    check_solution(got, ref, scene["projections"].shape[0], "mot_fresh30", fixed_pts=scene["pts"])


@pytest.mark.gpu
def test_point_on_principal_axis_stops_like_the_reference():
    """a projection at r = 0 is NaN; the solve ends through stop 7 (non-finite error) with the inputs unchanged"""
    scene = synth.ba_scene_fisheye(8, 200, 3, seed=5, ordinary_fraction=0.0)
    scene["c"][0] = scene["gt_c"][0]                  # camera 0 sits on the x axis with an exact axis-aligned rotation
    i = int(np.nonzero(scene["vmask"][:, 0])[0][0])
    scene["pts"][i] = 0.0                             # on camera 0's principal axis
    got = bundle.run_sfm(scene, optimize_for_fisheye=1, **fe(scene))
    assert int(got["info"][6]) == 7 and int(got["info"][5]) == 0
    assert np.array_equal(got["pts"], scene["pts"])
    from oracle import loader
    if loader.ref_sba() is not None:
        ref = loader.run_sfm_ref(scene, optimize_for_fisheye=1, **fe(scene))
        assert int(ref["info"][6]) == 7 and int(ref["info"][5]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fix_points", [0, 1])
def test_fe_entries_without_fisheye_equal_the_old_ones(fix_points):
    """optimize_for_fisheye = 0: bsfm_run_sfm_fe / _crs_fe are bit-identical to bsfm_run_sfm, also when cameras carry
    fisheye = 1 (the byte is not read then)"""
    scene = synth.ba_scene_fisheye(12, 800, 4, seed=7, known_fraction=0.25)
    kw = {"fix_points": fix_points}
    old = bundle.run_sfm(scene, **kw, **fe(scene))
    new = bundle.run_sfm(scene, optimize_for_fisheye=0, **kw, **fe(scene))
    new_crs = bundle.run_sfm(synth.crs_scene(scene), optimize_for_fisheye=0, **kw, **fe(scene))
    for key in ("R", "c", "f", "k", "pts", "info"):
        assert np.array_equal(old[key], new[key]), key
        assert np.array_equal(old[key], new_crs[key]), key
    if not fix_points:
        ex_old = bundle.run_sfm(scene, export=True, **fe(scene))
        ex_new = bundle.run_sfm(scene, optimize_for_fisheye=0, export=True, **fe(scene))
        for key in ("V", "S", "U", "W"):
            assert np.array_equal(ex_old[key], ex_new[key]), key


@pytest.mark.gpu
def test_old_entries_still_refuse_fisheye():
    """bsfm_run_sfm keeps returning BSFM_ERR_UNSUPPORTED for optimize_for_fisheye = 1, and bsfm_reprojection_outliers for
    fisheye cameras: callers may route that work elsewhere"""
    scene = synth.ba_scene_fisheye(6, 100, 3, seed=8)
    fn = getattr(bundle.load_library(), "bsfm_run_sfm")
    bundle._bind_run_sfm(fn)
    fn.argtypes = fn.argtypes + [ctypes.c_void_p]
    fn.restype = ctypes.c_int
    out = bundle.call_run_sfm(fn, scene, optimize_for_fisheye=1, extra_info=True, **fe(scene))
    assert out["rc"] == -6 and "fisheye" in last_error()
    with pytest.raises(BsfmError, match="fisheye"):
        bundle.reprojection_outliers(scene, **fe(scene))


def _export_normal_blocks(scene, cams, cnp, est_focal, undistort, jac_mode):
    """U, V, W of the Jacobian at the starting point through bsfm_sba_motstr_levmar_model_fe (itmax = 0: the export pass
    alone, sba_levmar.c:1633-2026)"""
    lib = bundle.load_library()
    fn = lib.bsfm_sba_motstr_levmar_model_fe
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_void_p,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_int]
    fn.restype = c.c_int
    n, m = scene["vmask"].shape
    p, cnp_ = bundle.pack_params(scene, est_focal, undistort)
    assert cnp_ == cnp
    R_init = np.ascontiguousarray(scene["R"], np.float64); f_fixed = np.ascontiguousarray(scene["f"], np.float64)
    model = bundle.SfmModel(est_focal, undistort, 1, 0.001, 5.0, R_init.ctypes.data, f_fixed.ctypes.data)
    vm = np.ascontiguousarray(scene["vmask"], np.int8); x = np.ascontiguousarray(scene["projections"]).reshape(-1).copy()
    opts = np.array([1.0e-3, 1.0e-10, 1e-12, 1.0e-12, 0.0, 4.0e-2]); info = np.zeros(10)
    V = np.zeros((n, 9)); S = np.zeros((m * cnp, m * cnp)); U = np.zeros((m, cnp * cnp)); W = np.zeros((m * cnp, 3 * n))
    rc = fn(n, m, 0, vm.ctypes.data, p.ctypes.data, cnp, 3, x.ctypes.data, None, 2, ctypes.addressof(model), jac_mode, 0, 0,
            opts.ctypes.data, info.ctypes.data, 0, None, 0, None, V.ctypes.data, S.ctypes.data, U.ctypes.data, W.ctypes.data,
            ctypes.addressof(cams), 1)
    assert rc == 0, rc
    return U.reshape(m, cnp, cnp), V.reshape(n, 3, 3), W


@pytest.mark.gpu
@pytest.mark.parametrize("est_focal,undistort", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_analytic_jacobian_blocks_match_finite_differences(est_focal, undistort):
    """the analytic Jacobian of the fisheye projection against forward differences, entry by entry through U, V and W,
    each entry scaled by the norms of its two Jacobian columns; the k columns are exactly zero in both modes.  Fisheye,
    ordinary and calibrated cameras are mixed."""
    scene = synth.ba_scene_fisheye(8, 120, 3, seed=9, ordinary_fraction=0.25, known_fraction=0.25)
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], np.tile([0.05, -0.02], (8, 1)), **fe(scene))
    cnp = 6 + est_focal + 2 * undistort
    Ua, Va, Wa = _export_normal_blocks(scene, cams, cnp, est_focal, undistort, 1)
    Uf, Vf, Wf = _export_normal_blocks(scene, cams, cnp, est_focal, undistort, 0)
    if undistort:
        kc = slice(6 + est_focal, 8 + est_focal)
        for U, W in ((Ua, Wa), (Uf, Wf)):
            assert not U[:, kc, :].any() and not U[:, :, kc].any()
            assert not W.reshape(8, cnp, -1)[:, kc, :].any()
    du = np.sqrt(np.maximum(np.diagonal(Uf, axis1=1, axis2=2), 1e-300))
    dv = np.sqrt(np.maximum(np.diagonal(Vf, axis1=1, axis2=2), 1e-300))
    assert np.array_equal(np.diagonal(Uf, axis1=1, axis2=2) == 0.0, np.diagonal(Ua, axis1=1, axis2=2) == 0.0)
    eu = np.abs(Ua - Uf) / (du[:, :, None] * du[:, None, :])
    ev = np.abs(Va - Vf) / (dv[:, :, None] * dv[:, None, :])
    ew = np.abs(Wa - Wf) / (du.reshape(-1)[:, None] * dv.reshape(-1)[None, :])
    assert eu.max() <= 2e-3, ("U", eu.max(), np.unravel_index(eu.argmax(), eu.shape))
    assert ev.max() <= 2e-3, ("V", ev.max())
    assert ew.max() <= 2e-3, ("W", ew.max())


@pytest.mark.gpu
def test_analytic_jacobian_reaches_fd_optimum(monkeypatch):
    g = gold()
    scene, kw, ref = gold_case(g, "mixed")
    monkeypatch.setenv("BSFM_BA_JAC", "analytic")
    got = bundle.run_sfm(scene, optimize_for_fisheye=1, **kw, **fe(scene))
    nvis = scene["projections"].shape[0]
    assert abs(np.sqrt(got["info"][1] / nvis) - np.sqrt(ref["info"][1] / nvis)) <= 2e-3
    assert abs(got["info"][0] - ref["info"][0]) <= 1e-9 * abs(ref["info"][0])


@pytest.mark.gpu
def test_levmar_model_fe_with_device_pointers():
    import torch
    g = gold()
    scene, kw, ref = gold_case(g, "mixed")
    p, cnp = bundle.pack_params(scene)
    n, m = scene["vmask"].shape
    d_vmask = torch.from_numpy(np.ascontiguousarray(scene["vmask"], np.int8)).cuda()
    d_p = torch.from_numpy(p.copy()).cuda()
    d_x = torch.from_numpy(np.ascontiguousarray(scene["projections"]).reshape(-1)).cuda()
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **fe(scene))
    torch.cuda.synchronize()
    its, info = bundle.levmar_model(n, m, d_vmask.data_ptr(), d_p.data_ptr(), d_x.data_ptr(), cnp, scene["R"], scene["f"],
                                    init_params=cams, optimize_for_fisheye=1)
    got = bundle.unpack_params(d_p.cpu().numpy(), scene)
    got["info"] = info
    assert its == int(info[5])
    check_solution(got, ref, scene["projections"].shape[0], "levmar_model_fe")
    with pytest.raises(BsfmError, match="init_params"):
        bundle.levmar_model(n, m, d_vmask.data_ptr(), d_p.data_ptr(), d_x.data_ptr(), cnp, scene["R"], scene["f"],
                            optimize_for_fisheye=1)


@pytest.mark.gpu
def test_mot_levmar_model_fe_host_pointers():
    g = gold()
    scene, kw, ref = gold_case(g, "fixpts")
    p, cnp = bundle.pack_params(scene)
    n, m = scene["vmask"].shape
    a = np.ascontiguousarray(p[:m * cnp])
    pts = np.ascontiguousarray(scene["pts"], np.float64)
    vm = np.ascontiguousarray(scene["vmask"], np.int8)
    x = np.ascontiguousarray(scene["projections"])
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **fe(scene))
    its, info = bundle.mot_levmar_model(n, m, vm.ctypes.data, a.ctypes.data, x.ctypes.data, pts.ctypes.data, cnp, scene["R"],
                                        scene["f"], init_params=cams, optimize_for_fisheye=1)
    got = bundle.unpack_params(np.concatenate([a, pts.reshape(-1)]), scene)
    got["info"] = info
    check_solution(got, ref, scene["projections"].shape[0], "mot_levmar_model_fe", fixed_pts=scene["pts"])


def _sba_call(sba, drv, scene, mot):
    n, m = scene["vmask"].shape
    p, cnp = bundle.pack_params(scene)
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **fe(scene))
    for j in range(m):
        cams[j].f_scale, cams[j].k_scale = 0.001, 5.0       # what run_sfm sets before it calls sba (sfm.c:652-696)
    pts = np.ascontiguousarray(scene["pts"], np.float64)
    glob = _globals(scene, cams, 1, 1, 1)
    glob.points = pts.ctypes.data
    vm = np.ascontiguousarray(scene["vmask"], np.int8)
    x = np.ascontiguousarray(scene["projections"]).reshape(-1).copy()
    opts = np.array([1.0e-3, 1.0e-10, 1e-12, 1.0e-12, 0.0, 4.0e-2])     # sfm.c:705-714
    info = np.zeros(10)
    V = ctypes.c_void_p
    if mot:
        fn = sba.sba_mot_levmar
        fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, V, V, ctypes.c_int, V, V, ctypes.c_int, V, V, V, ctypes.c_int,
                       ctypes.c_int, V, V, ctypes.c_int, V]
        proj = ctypes.cast(drv.sfm_project_point2_fisheye_mot, V).value
        a = np.ascontiguousarray(p[:m * cnp])
        rc = fn(n, m, 0, vm.ctypes.data, a.ctypes.data, cnp, x.ctypes.data, None, 2, proj, None, ctypes.addressof(glob), 150, 0,
                opts.ctypes.data, info.ctypes.data, 0, None)
        p = np.concatenate([a, pts.reshape(-1)])
    else:
        fn = sba.sba_motstr_levmar
        fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, V, V, ctypes.c_int, ctypes.c_int, V, V, ctypes.c_int, V, V, V,
                       ctypes.c_int, ctypes.c_int, V, V, ctypes.c_int, V, ctypes.c_int, V, V, V, V, V]
        proj = ctypes.cast(drv.sfm_project_point2_fisheye, V).value
        rc = fn(n, m, 0, vm.ctypes.data, p.ctypes.data, cnp, 3, x.ctypes.data, None, 2, proj, None, ctypes.addressof(glob), 150, 0,
                opts.ctypes.data, info.ctypes.data, 0, None, 0, None, None, None, None, None)
    fn.restype = ctypes.c_int
    return rc, info, p


@pytest.mark.gpu
@pytest.mark.parametrize("mot", [0, 1])
def test_sba_drop_in_accepts_fisheye_callbacks(mot):
    """sba_motstr_levmar / sba_mot_levmar of libsba_b200.so, called with the reference signature and the exported
    sfm_project_point2_fisheye(_mot), give what bsfm_run_sfm_fe gives"""
    drv = _sfmdrv()
    sba = ctypes.CDLL(os.path.join(SHIM, "libsba_b200.so"))
    g = gold()
    scene, kw, ref = gold_case(g, "fixpts" if mot else "mixed")
    rc, info, p = _sba_call(sba, drv, scene, mot)
    got_run = bundle.run_sfm(scene, optimize_for_fisheye=1, fix_points=mot, **fe(scene))
    assert rc == int(got_run["info"][5]) == int(info[5])
    assert np.array_equal(info[:7], got_run["info"][:7])
    got = bundle.unpack_params(p, scene)
    for key in ("R", "c", "f", "k", "pts"):
        assert np.allclose(got[key], got_run[key], rtol=1e-12, atol=1e-12), key


@pytest.mark.gpu
@pytest.mark.parametrize("crs", [0, 1])
def test_outlier_pass_fe_equals_golden(crs):
    g = gold()
    sc = {k: g[f"outl_{k}"] for k in SCENE_KEYS if f"outl_{k}" in g.files}
    lo, hi = g["outl_thresholds"]
    src = synth.crs_scene(sc) if crs else sc
    got = bundle.reprojection_outliers(src, 1, float(lo), float(hi), g["outl_protected"], optimize_for_fisheye=1, **fe(sc))
    assert np.allclose(got["dist"], g["outl_ref_dist"], rtol=1e-12, atol=1e-12)
    assert np.array_equal(got["stats"][:, 0], g["outl_ref_stats"][:, 0])
    assert np.allclose(got["stats"][:, 1:], g["outl_ref_stats"][:, 1:], rtol=1e-12, atol=1e-12, equal_nan=True)
    assert np.array_equal(got["outliers"], g["outl_ref_outliers"])
    assert np.allclose(got["errors"], g["outl_ref_errors"], rtol=1e-12)
    assert abs(got["global_mean"] - float(g["outl_ref_global_mean"])) <= 1e-12 * abs(float(g["outl_ref_global_mean"]))


@pytest.mark.gpu
def test_outlier_pass_fe_without_fisheye_equals_old_entry():
    """optimize_for_fisheye = 0: fisheye cameras are projected as ordinary ones, bit for bit what the old entry gives"""
    g = gold()
    sc = {k: g[f"outl_{k}"] for k in SCENE_KEYS if f"outl_{k}" in g.files}
    lo, hi = g["outl_thresholds"]
    new = bundle.reprojection_outliers(sc, 1, float(lo), float(hi), g["outl_protected"], optimize_for_fisheye=0, **fe(sc))
    old = bundle.reprojection_outliers(dict(sc), 1, float(lo), float(hi), g["outl_protected"])
    for key in ("dist", "stats", "outliers", "errors"):
        assert np.array_equal(new[key], old[key], equal_nan=key == "stats"), key
    assert new["global_mean"] == old["global_mean"]
