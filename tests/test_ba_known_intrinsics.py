"""Bundle adjustment of calibrated cameras (camera_params_t::known_intrinsics with K_known / k_known,
lib/sfm-driver/sfm.c:339-357; what `bundler --intrinsics` sets up, src/Bundle.cpp:241-247).

CPU tests pin the committed outputs of the unmodified reference (tests/golden/ba_known_intrinsics_golden.npz, made by
tests/golden/make_ba_known_intrinsics_golden.py) and the host sfm_project_point3 of the run_sfm shim against a numpy
restatement of the projection.  GPU tests run every golden case through bsfm_run_sfm and the other entry points.

Tolerances as in tests/test_ba_gpu.py: final reprojection RMSE within 1e-5 px, same iteration count and stop reason
(motion-only: a rounding-driven stop, see check_solution), parameters within 1e-4 of each group's largest magnitude,
initial error within 1e-9 relative."""
import ctypes
import os

import numpy as np
import pytest

from bundler_sfm_b200 import bundle, synth
from tests.ba_restatement import port_run_sfm     # numpy restatement of run_sfm, with the calibrated branch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ba_known_intrinsics_golden.npz")
SHIM = os.path.join(ROOT, "shim", "_build")
SCENE_KEYS = ("vmask", "projections", "R", "c", "f", "k", "pts", "known", "K_known", "k_known")
SOLVE_CASES = ("ef0_ud0", "ef0_ud1", "ef1_ud0", "ef1_ud1", "mixed", "cons", "fixpts", "tcam")
RMSE_TOL = 1e-5
PARAM_TOL = 1e-4


# ---- numpy restatement of sfm_project_rd (sfm.c:302-380), scalar, in the reference's operation order -----------------
def project_ref(R, dt, b, f, k_rad, undistort, explicit_centers, known, K, kk):
    if explicit_centers:
        b2 = (b[0] - dt[0], b[1] - dt[1], b[2] - dt[2])
        bc = [R[0] * b2[0] + R[1] * b2[1] + R[2] * b2[2], R[3] * b2[0] + R[4] * b2[1] + R[5] * b2[2],
              R[6] * b2[0] + R[7] * b2[1] + R[8] * b2[2]]
    else:
        bc = [R[0] * b[0] + R[1] * b[1] + R[2] * b[2], R[3] * b[0] + R[4] * b[1] + R[5] * b[2],
              R[6] * b[0] + R[7] * b[1] + R[8] * b[2]]
        bc = [bc[0] + dt[0], bc[1] + dt[1], bc[2] + dt[2]]
    if not known:
        p0 = -bc[0] * f / bc[2]
        p1 = -bc[1] * f / bc[2]
    else:
        x_n = -bc[0] / bc[2]
        y_n = -bc[1] / bc[2]
        rsq = x_n * x_n + y_n * y_n
        factor = 1.0 + kk[0] * rsq + kk[1] * rsq * rsq + kk[4] * rsq * rsq * rsq
        dx_x = 2 * kk[2] * x_n * y_n + kk[3] * (rsq + 2 * x_n * x_n)
        dx_y = kk[2] * (rsq + 2 * y_n * y_n) + 2 * kk[3] * x_n * y_n
        x_d = x_n * factor + dx_x
        y_d = y_n * factor + dx_y
        p0 = K[0] * x_d + K[1] * y_d + K[2]
        p1 = K[4] * y_d + K[5]
    if undistort:
        rsq = (p0 * p0 + p1 * p1) / (f * f)
        factor = 1.0 + k_rad[0] * rsq + k_rad[1] * rsq * rsq
        p0 *= factor
        p1 *= factor
    return p0, p1


def rot_update(R, w):      # sfm.c:77-116
    th = np.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    R = np.asarray(R, float).reshape(3, 3)
    if th == 0.0:
        return R.reshape(9)
    nx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
    return ((np.eye(3) + nx * np.sin(th) + nx @ nx * (1.0 - np.cos(th))) @ R).reshape(9)


def gold():
    return np.load(GOLD)


def gold_case(g, name):
    scene = {k: g[f"{name}_{k}"] for k in SCENE_KEYS}
    kw = {k[len(name) + 4:]: g[k].item() for k in g.files if k.startswith(f"{name}_kw_")}
    for k in ("constrained", "constraints", "weights", "points_constraints"):
        if f"{name}_{k}" in g.files:
            kw[k] = g[f"{name}_{k}"]
    ref = {k: g[f"{name}_ref_{k}"] for k in ("R", "c", "f", "k", "pts", "info")}
    return scene, kw, ref


def ki(scene):
    return {"known": scene["known"], "K_known": scene["K_known"], "k_known": scene["k_known"]}


def rel_group_err(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def check_solution(got, ref, nvis, what, fixed_pts=None, known=None, est_focal=1, undistort=1):
    r_gpu, r_ref = np.sqrt(got["info"][1] / nvis), np.sqrt(ref["info"][1] / nvis)
    assert abs(r_gpu - r_ref) <= RMSE_TOL, (what, r_gpu, r_ref)
    if fixed_pts is None:
        assert int(got["info"][5]) == int(ref["info"][5]), (what, "iterations", got["info"][5], ref["info"][5])
        assert int(got["info"][6]) == int(ref["info"][6]), (what, "stop reason", got["info"][6], ref["info"][6])
    else:
        # motion-only solves stop through rule 4 with eps4 = 0, i.e. when  pdp - 2 sqrt(p pdp) < -p  holds by ROUNDING at
        # convergence (sba_levmar.c:2596), or through rule 2: the iteration at which that happens is not a property of the
        # algorithm, so only the converged solution is compared (as in tests/test_ba_gpu.py, whose scenes stop sooner)
        assert int(got["info"][6]) in (2, 4), (what, "stop reason", got["info"][6])
    for key in ("R", "c", "pts"):
        err = rel_group_err(got[key], ref[key])
        assert err <= PARAM_TOL, (what, key, err)
    # A calibrated camera's focal parameter only enters through the radial step, which depends on k1 / f^2 and k2 / f^4
    # alone: with est_focal_length and undistort, (f, k1, k2) has an exact null direction, and where along it a solve ends depends on the
    # damping path and on rounding.  Those cameras are compared through the radial factor they define at 250 px, a
    # dimensionless number held to the parameter tolerance (the reprojection RMSE above stays the tight check).
    fk = np.zeros(len(got["f"]), bool) if known is None or not (est_focal and undistort) else np.asarray(known) != 0
    if (~fk).any():
        assert rel_group_err(got["f"][~fk], ref["f"][~fk]) <= PARAM_TOL, (what, "f", rel_group_err(got["f"][~fk], ref["f"][~fk]))
        assert np.max(np.abs(got["k"][~fk] - ref["k"][~fk])) * 5.0 <= PARAM_TOL * max(1.0, 5.0 * np.max(np.abs(ref["k"][~fk]))), (what, "k")
    if fk.any():
        def radial(sol):
            s2 = (250.0 / sol["f"][fk]) ** 2
            return sol["k"][fk, 0] * s2 + sol["k"][fk, 1] * s2 * s2
        assert np.max(np.abs(radial(got) - radial(ref))) <= PARAM_TOL, (what, "radial factor", np.max(np.abs(radial(got) - radial(ref))))
    assert abs(got["info"][0] - ref["info"][0]) <= 1e-9 * abs(ref["info"][0]), (what, "initial error")
    if fixed_pts is not None:
        assert np.array_equal(got["pts"], fixed_pts), (what, "points must stay fixed")


# ---- CPU: the golden file against the numpy restatement -------------------------------------------------------------
@pytest.mark.parametrize("name", ["ef0_ud0", "ef0_ud1", "ef1_ud0", "ef1_ud1", "mixed", "fixpts"])
def test_golden_errors_match_numpy_projection(name):
    """the reference's initial and final errors (info[0], info[1]) are the squared reprojection errors of the stored
    scene and solution under the calibrated-camera projection: pins what the golden file was made with"""
    g = gold()
    scene, kw, ref = gold_case(g, name)
    nvis = scene["projections"].shape[0]
    ud = kw.get("undistort", 1)
    k0 = scene["k"] if ud else np.zeros_like(scene["k"])
    init = dict(scene, k=k0)
    sol = dict(ref, k=ref["k"] if ud else np.zeros_like(ref["k"]))
    r0 = bundle.reprojection_rmse(scene, init, **ki(scene))
    r1 = bundle.reprojection_rmse(scene, sol, **ki(scene))
    assert abs(r0 - np.sqrt(ref["info"][0] / nvis)) <= 1e-9 * r0, (name, r0)
    assert abs(r1 - np.sqrt(ref["info"][1] / nvis)) <= 1e-9 * r1, (name, r1)
    # and the calibration is what made the difference: ignoring it leaves a far larger error
    assert bundle.reprojection_rmse(scene, sol) > 2.0 * r1


@pytest.mark.parametrize("name", ["ef0_ud0", "ef0_ud1", "ef1_ud0", "ef1_ud1", "mixed", "cons", "tcam"])
def test_cpu_restatement_reproduces_golden(name):
    """the numpy restatement of run_sfm above, with the calibrated branch, reproduces the unmodified reference's outputs:
    same iterations and stop reason, RMSE within 1e-5 px, parameters within 1e-4, initial error within 1e-9"""
    g = gold()
    scene, kw, ref = gold_case(g, name)
    got = port_run_sfm(scene, **kw, **ki(scene))
    assert got is not None
    check_solution(got, ref, scene["projections"].shape[0], "port_" + name, known=scene["known"],
                   est_focal=kw.get("est_focal_length", 1), undistort=kw.get("undistort", 1))


def test_golden_outlier_pass_matches_numpy_restatement():
    """distances / per-camera statistics / outliers of the golden outlier case (src/Bundle.cpp:659-856) restated"""
    g = gold()
    sc = {k: g[f"outl_{k}"] for k in SCENE_KEYS}
    prot = g["outl_protected"]
    lo, hi = g["outl_thresholds"]
    vm = sc["vmask"] != 0
    obs_pt, obs_cam = np.nonzero(vm)
    dist = np.empty(len(obs_pt))
    for o, (i, j) in enumerate(zip(obs_pt, obs_cam)):
        p0, p1 = project_ref(sc["R"][j], sc["c"][j], sc["pts"][i], sc["f"][j], sc["k"][j], 1, 1, sc["known"][j],
                             sc["K_known"][j], sc["k_known"][j])
        dx, dy = p0 - sc["projections"][o, 0], p1 - sc["projections"][o, 1]
        dist[o] = np.sqrt(dx * dx + dy * dy)
    assert np.allclose(dist, g["outl_ref_dist"], rtol=1e-12, atol=1e-12)
    first = {}
    stats = np.zeros((vm.shape[1], 5))
    for j in range(vm.shape[1]):
        d = dist[obs_cam == j]
        n = len(d)
        k80, k50 = int(0.8 * n + 0.5), int(0.5 * n + 0.5)                 # iround, lib/imagelib/util.c:75-81
        med80 = np.sort(d)[k80] if k80 < n else 0.0                        # kth_element_copy, qsort.c:152-204
        med50 = np.sort(d)[k50] if k50 < n else 0.0
        thresh = min(max(1.2 * 2.0 * med80, lo), hi)                       # Bundle.cpp:761-771
        stats[j] = (n, np.sum(d) / n, med50, med80, thresh)
        for i, v in zip(obs_pt[obs_cam == j], d):
            if v > thresh and not prot[i] and i not in first:
                first[i] = (j, v)
    assert np.array_equal(stats[:, 0], g["outl_ref_stats"][:, 0])
    assert np.allclose(stats[:, 1:], g["outl_ref_stats"][:, 1:], rtol=1e-12, atol=1e-12)
    order = sorted(first, key=lambda i: (first[i][0], i))
    assert np.array_equal(np.array(order, np.int32), g["outl_ref_outliers"])
    assert np.allclose([first[i][1] for i in order], g["outl_ref_errors"], rtol=1e-12)
    assert len(order) > 0 and not any(prot[i] for i in order)


# ---- CPU: the host sfm_project_point3 of libsfmdrv_b200.so ----------------------------------------------------------
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
    lib.sfm_project_point3.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.sfm_project_point3.restype = None
    return lib


@pytest.mark.parametrize("est_focal,undistort", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("explicit_centers", [1, 0])
def test_shim_host_projection_matches_numpy(est_focal, undistort, explicit_centers):
    lib = _sfmdrv()
    sc = synth.ba_scene_known_intrinsics(8, 50, 3, seed=3, ordinary_fraction=0.5)
    m = len(sc["f"])
    rng = np.random.default_rng(est_focal * 2 + undistort)
    k_rad = rng.uniform(-0.05, 0.05, (m, 2))
    cams = bundle.make_cameras(sc["R"], sc["c"], sc["f"], k_rad, **ki(sc))
    for j in range(m):
        cams[j].f_scale, cams[j].k_scale = 0.001, 5.0
    g = SfmGlobal()
    g.num_cameras, g.num_points = m, sc["pts"].shape[0]
    g.num_params_per_camera = 6 + est_focal + 2 * undistort
    g.est_focal_length, g.explicit_camera_centers, g.estimate_distortion = est_focal, explicit_centers, undistort
    g.init_params = ctypes.addressof(cams)
    assert sorted(set(sc["known"].tolist())) == [0, 1]
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
            b = sc["pts"][i].copy()
            out = np.zeros(2)
            lib.sfm_project_point3(j, i, a.ctypes.data, b.ctypes.data, out.ctypes.data, ctypes.addressof(g))
            f = a[6] / 0.001 if est_focal else sc["f"][j]
            kr = a[6 + est_focal:8 + est_focal] / 5.0 if undistort else None
            want = project_ref(rot_update(sc["R"][j], w), dt, b, f, kr, undistort, explicit_centers, sc["known"][j],
                               sc["K_known"][j], sc["k_known"][j])
            worst = max(worst, float(np.max(np.abs(out - np.array(want)) / np.maximum(np.abs(want), 1.0))))
    assert worst <= 1e-12, worst


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", SOLVE_CASES)
def test_golden_cases_through_run_sfm(name):
    g = gold()
    scene, kw, ref = gold_case(g, name)
    got = bundle.run_sfm(scene, **kw, **ki(scene))
    check_solution(got, ref, scene["projections"].shape[0], name, fixed_pts=scene["pts"] if kw.get("fix_points") else None,
                   known=scene["known"], est_focal=kw.get("est_focal_length", 1), undistort=kw.get("undistort", 1))


def _ref_or_skip():
    from oracle import loader
    if loader.ref_sba() is None:
        pytest.skip("oracle/_ref/libref_sba.so not available (oracle.run_sfm_oracle's C restatement has no calibrated-camera "
                    "branch; port_run_sfm of tests/ba_restatement.py is pinned to the golden file instead)")
    return loader


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,kw", [
    (20, 2000, {}),
    (16, 1500, {"est_focal_length": 0, "undistort": 1}),
    (240, 4000, {"undistort": 0}),     # cnp = 7: reduced system 1680 > 1536 unknowns -> the large Cholesky path
])
def test_fresh_scene_vs_reference(m, n, kw):
    loader = _ref_or_skip()
    scene = synth.ba_scene_known_intrinsics(m, n, 5, seed=m + 1, ordinary_fraction=0.25)
    got = bundle.run_sfm(scene, **kw, **ki(scene))
    ref = loader.run_sfm_ref(scene, **kw, **ki(scene))
    check_solution(got, ref, scene["projections"].shape[0], f"fresh{m}", known=scene["known"],
                   est_focal=kw.get("est_focal_length", 1), undistort=kw.get("undistort", 1))
    assert got["info"][1] < 0.1 * got["info"][0]


@pytest.mark.gpu
def test_motion_only_fresh_scene_vs_reference():
    loader = _ref_or_skip()
    scene = synth.ba_scene_known_intrinsics(30, 3000, 5, seed=41, ordinary_fraction=0.3)
    got = bundle.run_sfm(scene, fix_points=1, **ki(scene))
    ref = loader.run_sfm_ref(scene, fix_points=1, **ki(scene))
    check_solution(got, ref, scene["projections"].shape[0], "mot_fresh30", fixed_pts=scene["pts"], known=scene["known"])


@pytest.mark.gpu
def test_levmar_model_ki_with_device_pointers():
    """bsfm_sba_motstr_levmar_model_ki on device-resident vmask / p / x gives the run_sfm solution"""
    import torch
    g = gold()
    scene, kw, ref = gold_case(g, "mixed")
    p, cnp = bundle.pack_params(scene)
    n, m = scene["vmask"].shape
    d_vmask = torch.from_numpy(np.ascontiguousarray(scene["vmask"], np.int8)).cuda()
    d_p = torch.from_numpy(p.copy()).cuda()
    d_x = torch.from_numpy(np.ascontiguousarray(scene["projections"]).reshape(-1)).cuda()
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **ki(scene))
    torch.cuda.synchronize()
    its, info = bundle.levmar_model(n, m, d_vmask.data_ptr(), d_p.data_ptr(), d_x.data_ptr(), cnp, scene["R"], scene["f"],
                                    init_params=cams)
    got = bundle.unpack_params(d_p.cpu().numpy(), scene)
    got["info"] = info
    assert its == int(info[5])
    check_solution(got, ref, scene["projections"].shape[0], "levmar_model_ki", known=scene["known"])
    # without the calibration the same entry point solves a different problem
    its2, info2 = bundle.levmar_model(n, m, d_vmask.data_ptr(), torch.from_numpy(p.copy()).cuda().data_ptr(), d_x.data_ptr(), cnp,
                                      scene["R"], scene["f"])
    assert info2[0] > 2.0 * info[0]


@pytest.mark.gpu
def test_mot_levmar_model_ki_host_pointers():
    g = gold()
    scene, kw, ref = gold_case(g, "fixpts")
    p, cnp = bundle.pack_params(scene)
    n, m = scene["vmask"].shape
    a = np.ascontiguousarray(p[:m * cnp])
    pts = np.ascontiguousarray(scene["pts"], np.float64)
    vm = np.ascontiguousarray(scene["vmask"], np.int8)
    x = np.ascontiguousarray(scene["projections"])
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **ki(scene))
    its, info = bundle.mot_levmar_model(n, m, vm.ctypes.data, a.ctypes.data, x.ctypes.data, pts.ctypes.data, cnp, scene["R"], scene["f"],
                                        init_params=cams)
    got = bundle.unpack_params(np.concatenate([a, pts.reshape(-1)]), scene)
    got["info"] = info
    check_solution(got, ref, scene["projections"].shape[0], "mot_levmar_model_ki", fixed_pts=scene["pts"], known=scene["known"])


@pytest.mark.gpu
def test_sba_drop_in_with_calibrated_cameras():
    """sba_motstr_levmar of libsba_b200.so, called with the reference signature, sfm_project_point3 of libsfmdrv_b200.so
    and an sfm_global_t of calibrated cameras, gives what bsfm_run_sfm gives"""
    drv = _sfmdrv()
    sba = ctypes.CDLL(os.path.join(SHIM, "libsba_b200.so"))
    g = gold()
    scene, kw, ref = gold_case(g, "mixed")
    n, m = scene["vmask"].shape
    p, cnp = bundle.pack_params(scene)
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **ki(scene))
    for j in range(m):
        cams[j].f_scale, cams[j].k_scale = 0.001, 5.0       # what run_sfm sets before it calls sba (sfm.c:652-696)
    glob = SfmGlobal()
    glob.num_cameras, glob.num_points, glob.num_params_per_camera = m, n, cnp
    glob.est_focal_length, glob.explicit_camera_centers, glob.estimate_distortion = 1, 1, 1
    glob.init_params = ctypes.addressof(cams)
    vm = np.ascontiguousarray(scene["vmask"], np.int8)
    x = np.ascontiguousarray(scene["projections"]).reshape(-1).copy()
    opts = np.array([1.0e-3, 1.0e-10, 1e-12, 1.0e-12, 0.0, 4.0e-2])     # sfm.c:705-714
    info = np.zeros(10)
    fn = sba.sba_motstr_levmar
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                   ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    proj = ctypes.cast(drv.sfm_project_point3, ctypes.c_void_p).value
    rc = fn(n, m, 0, vm.ctypes.data, p.ctypes.data, cnp, 3, x.ctypes.data, None, 2, proj, None, ctypes.addressof(glob), 150, 0,
            opts.ctypes.data, info.ctypes.data, 0, None, 0, None, None, None, None, None)
    got_run = bundle.run_sfm(scene, **ki(scene))
    assert rc == int(got_run["info"][5]) == int(info[5])
    assert np.array_equal(info[:7], got_run["info"][:7])
    got = bundle.unpack_params(p, scene)      # numpy unpacking: rounds differently from run_sfm's C unpacking
    for key in ("R", "c", "f", "k", "pts"):
        assert np.allclose(got[key], got_run[key], rtol=1e-12, atol=1e-12), key


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ef1_ud1", "ef0_ud0", "mixed"])
def test_analytic_jacobian_reaches_fd_optimum(name, monkeypatch):
    g = gold()
    scene, kw, ref = gold_case(g, name)
    monkeypatch.setenv("BSFM_BA_JAC", "analytic")
    got = bundle.run_sfm(scene, **kw, **ki(scene))
    nvis = scene["projections"].shape[0]
    assert abs(np.sqrt(got["info"][1] / nvis) - np.sqrt(ref["info"][1] / nvis)) <= 2e-3, name
    assert abs(got["info"][0] - ref["info"][0]) <= 1e-9 * abs(ref["info"][0])


def _export_normal_blocks(scene, cams, cnp, est_focal, undistort, jac_mode):
    """U (m x cnp x cnp), V (n x 3 x 3) and W ((m cnp) x 3n) of the Jacobian at the starting point: itmax = 0 skips the LM
    loop and the export pass (sba_levmar.c:1633-2026) forms them from one Jacobian evaluation in the chosen mode"""
    lib = bundle.load_library()
    fn = lib.bsfm_sba_motstr_levmar_model_ki
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_void_p,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p]
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
            ctypes.addressof(cams))
    assert rc == 0, rc
    return U.reshape(m, cnp, cnp), V.reshape(n, 3, 3), W


@pytest.mark.gpu
@pytest.mark.parametrize("est_focal,undistort", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_analytic_jacobian_blocks_match_finite_differences(est_focal, undistort):
    """the analytic Jacobian of calibrated cameras against forward differences, entry by entry through U = sum A^T A,
    V = sum B^T B and W = A^T B, each entry scaled by the norms of its two Jacobian columns.  The calibrated cameras have
    skew, an off-centre principal point, nonzero k4 and tangential terms large enough that dropping either one fails the
    check, and a nonzero radial pair so that the focal column is exercised; half of the cameras are ordinary ones."""
    scene = synth.ba_scene_known_intrinsics(6, 80, 3, seed=9, ordinary_fraction=0.5)
    m = len(scene["f"])
    kk = scene["k_known"].copy()
    kk[:, 2], kk[:, 3], kk[:, 4] = 0.02, -0.015, 0.01
    scene["K_known"][:, 1] = 3.0
    scene["k"] = np.tile([0.05, -0.02], (m, 1))
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], known=scene["known"], K_known=scene["K_known"], k_known=kk)
    cnp = 6 + est_focal + 2 * undistort
    Ua, Va, Wa = _export_normal_blocks(scene, cams, cnp, est_focal, undistort, 1)
    Uf, Vf, Wf = _export_normal_blocks(scene, cams, cnp, est_focal, undistort, 0)
    du = np.sqrt(np.maximum(np.diagonal(Uf, axis1=1, axis2=2), 1e-300))          # column norms, m x cnp
    dv = np.sqrt(np.maximum(np.diagonal(Vf, axis1=1, axis2=2), 1e-300))          # n x 3
    zero_cols = np.diagonal(Uf, axis1=1, axis2=2) == 0.0                        # focal column of a calibrated camera without undistort
    assert np.array_equal(zero_cols, np.diagonal(Ua, axis1=1, axis2=2) == 0.0)
    if est_focal and not undistort:
        assert zero_cols[scene["known"] != 0, 6].all()
    eu = np.abs(Ua - Uf) / (du[:, :, None] * du[:, None, :])
    ev = np.abs(Va - Vf) / (dv[:, :, None] * dv[:, None, :])
    ew = np.abs(Wa - Wf) / (du.reshape(-1)[:, None] * dv.reshape(-1)[None, :])
    assert eu.max() <= 2e-3, ("U", eu.max(), np.unravel_index(eu.argmax(), eu.shape))
    assert ev.max() <= 2e-3, ("V", ev.max())
    assert ew.max() <= 2e-3, ("W", ew.max())


@pytest.mark.gpu
def test_outlier_pass_equals_golden():
    g = gold()
    sc = {k: g[f"outl_{k}"] for k in SCENE_KEYS}
    lo, hi = g["outl_thresholds"]
    got = bundle.reprojection_outliers(sc, 1, float(lo), float(hi), g["outl_protected"], **ki(sc))
    assert np.allclose(got["dist"], g["outl_ref_dist"], rtol=1e-12, atol=1e-12)
    assert np.array_equal(got["stats"][:, 0], g["outl_ref_stats"][:, 0])
    assert np.allclose(got["stats"][:, 1:], g["outl_ref_stats"][:, 1:], rtol=1e-12, atol=1e-12, equal_nan=True)
    assert np.array_equal(got["outliers"], g["outl_ref_outliers"])
    assert np.allclose(got["errors"], g["outl_ref_errors"], rtol=1e-12)
    assert abs(got["global_mean"] - float(g["outl_ref_global_mean"])) <= 1e-12 * abs(float(g["outl_ref_global_mean"]))
