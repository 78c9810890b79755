"""Host-side mirror of the reference BA interface on top of the C ABI.

Reference (file:line under /root/reference):
  run_sfm(num_pts, num_cameras, ncons, vmask, projections, est_focal_length, const_focal_length,
          undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints,
          use_point_constraints, points_constraints, point_constraint_weight, fix_points,
          optimize_for_fisheye, eps2, Vout, Sout, Uout, Wout)          lib/sfm-driver/sfm.h:68-86
  camera_params_t                                                       lib/sfm-driver/sfm.h:32-51
"""
import ctypes

import numpy as np

from ._lib import load_library, check

NUM_CAMERA_PARAMS = 9


class CameraParams(ctypes.Structure):
    """== camera_params_t (lib/sfm-driver/sfm.h:32-51) / bsfm_camera_params_t"""
    _fields_ = [
        ("R", ctypes.c_double * 9), ("t", ctypes.c_double * 3), ("f", ctypes.c_double), ("k", ctypes.c_double * 2),
        ("k_inv", ctypes.c_double * 6), ("constrained", ctypes.c_char * NUM_CAMERA_PARAMS),
        ("constraints", ctypes.c_double * NUM_CAMERA_PARAMS), ("weights", ctypes.c_double * NUM_CAMERA_PARAMS),
        ("K_known", ctypes.c_double * 9), ("k_known", ctypes.c_double * 5), ("fisheye", ctypes.c_char),
        ("known_intrinsics", ctypes.c_char), ("f_cx", ctypes.c_double), ("f_cy", ctypes.c_double),
        ("f_rad", ctypes.c_double), ("f_angle", ctypes.c_double), ("f_focal", ctypes.c_double),
        ("f_scale", ctypes.c_double), ("k_scale", ctypes.c_double),
    ]


def make_cameras(R, c, f, k, constrained=None, constraints=None, weights=None, known=None, K_known=None, k_known=None,
                 fisheye=None, fisheye_params=None):
    """camera_params_t array.  known (m flags), K_known (m x 9) and k_known (m x 5) describe calibrated cameras
    (known_intrinsics, lib/sfm-driver/sfm.c:339-357); without them every camera is an ordinary one.  fisheye (m flags)
    and fisheye_params (m x 5: f_cx, f_cy, f_rad, f_angle, f_focal) fill the fisheye fields (src/Bundle.cpp:234-239),
    which only the fisheye projection reads (optimize_for_fisheye)."""
    m = len(f)
    cams = (CameraParams * m)()
    for j in range(m):
        cams[j].R[:] = list(np.asarray(R[j], float).reshape(9))
        cams[j].t[:] = list(np.asarray(c[j], float))
        cams[j].f = float(f[j])
        cams[j].k[:] = list(np.asarray(k[j], float))
        cams[j].f_scale = 1.0
        cams[j].k_scale = 1.0
        if constrained is not None:
            ctypes.memmove(ctypes.addressof(cams[j]) + CameraParams.constrained.offset,
                           bytes(bytearray(int(v) for v in constrained[j])), NUM_CAMERA_PARAMS)
            cams[j].constraints[:] = list(np.asarray(constraints[j], float))
            cams[j].weights[:] = list(np.asarray(weights[j], float))
        if known is not None and known[j]:
            cams[j].known_intrinsics = b"\x01"
            cams[j].K_known[:] = list(np.asarray(K_known[j], float).reshape(9))
            cams[j].k_known[:] = list(np.asarray(k_known[j], float).reshape(5))
        if fisheye is not None and fisheye[j]:
            cams[j].fisheye = b"\x01"
        if fisheye_params is not None:
            (cams[j].f_cx, cams[j].f_cy, cams[j].f_rad, cams[j].f_angle, cams[j].f_focal) = (float(v) for v in fisheye_params[j])
    return cams


def cameras_to_arrays(cams):
    m = len(cams)
    R = np.array([list(cams[j].R) for j in range(m)])
    c = np.array([list(cams[j].t) for j in range(m)])
    f = np.array([cams[j].f for j in range(m)])
    k = np.array([list(cams[j].k) for j in range(m)])
    return R, c, f, k


def _bind_run_sfm(fn):
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_int,
                   c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_double, c.c_int, c.c_int, c.c_double,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p]
    return fn


def _visibility_args(scene):
    """the visibility arguments of a scene dict for the C entries -> (n, m, args, keep-alive).  A dense scene passes
    [vmask] (n x m); a CRS scene (synth.crs_scene) passes [vis_ptr, vis_cam, nvis] to the _crs entries, with n = len(pts)
    and m = len(R).  vis_ptr / vis_cam may be numpy arrays or int32 torch tensors (pageable, pinned or CUDA memory: their
    own pointers are passed); an optional "nvis" entry declares a count other than len(vis_cam)."""
    if "vis_ptr" not in scene:
        vmask = np.ascontiguousarray(scene["vmask"], dtype=np.int8)
        n, m = vmask.shape
        return n, m, [vmask.ctypes.data], [vmask]
    ptrs, keep = [], []
    for key in ("vis_ptr", "vis_cam"):
        a = scene[key]
        if hasattr(a, "data_ptr"):
            assert str(a.dtype) == "torch.int32" and a.is_contiguous(), key
            ptrs.append(a.data_ptr() or None)
        else:
            a = np.ascontiguousarray(a, dtype=np.int32)
            ptrs.append(a.ctypes.data)
        keep.append(a)
    nvis = int(scene.get("nvis", len(scene["vis_cam"])))
    return len(scene["pts"]), len(scene["R"]), ptrs + [nvis], keep


def observations(scene):
    """(point, camera) of every observation of a dense or CRS scene, in the order of `projections`"""
    if "vis_ptr" in scene:
        ptr = np.asarray(scene["vis_ptr"], dtype=np.int64)
        return np.repeat(np.arange(len(ptr) - 1), np.diff(ptr)), np.asarray(scene["vis_cam"], dtype=np.int64)
    return np.nonzero(scene["vmask"])


def call_run_sfm(fn, scene, est_focal_length=1, undistort=1, explicit_camera_centers=1, ncons=0, eps2=1e-12,
                 use_constraints=0, constrained=None, constraints=None, weights=None,
                 use_point_constraints=0, points_constraints=None, point_constraint_weight=0.0,
                 extra_info=False, export=False, fix_points=0, known=None, K_known=None, k_known=None,
                 fisheye=None, fisheye_params=None, optimize_for_fisheye=0):
    """Calls a run_sfm-shaped C function (ours or the reference's) on a scene dict (synth.ba_scene), or
    bsfm_run_sfm_crs on a CRS scene (synth.crs_scene).  known / K_known / k_known: calibrated cameras, fisheye /
    fisheye_params: fisheye cameras (see make_cameras); optimize_for_fisheye is passed to the callee.
    Returns a dict with the refined R, c, f, k, pts (+ info when the callee provides it)."""
    n, m, vis_args, _keep = _visibility_args(scene)
    proj = np.ascontiguousarray(scene["projections"], dtype=np.float64)
    cams = make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], constrained, constraints, weights, known, K_known, k_known,
                        fisheye, fisheye_params)
    pts = np.ascontiguousarray(scene["pts"], dtype=np.float64).copy()
    pc = None
    if use_point_constraints:
        pc = np.ascontiguousarray(points_constraints, dtype=np.float64)
    cnp = 6 + (1 if est_focal_length else 0) + (2 if undistort else 0)
    ex = {}
    export_keys = "VSUW" if export is True else (export or "")
    if export:   # Vout, Sout, Uout, Wout (sba_levmar.c:1633-2026)
        ex = {"V": np.zeros((n, 9)), "S": np.zeros((m * cnp, m * cnp)), "U": np.zeros((m, cnp * cnp)), "W": np.zeros((m * cnp, 3 * n))}
    args = [n, m, ncons, *vis_args, proj.ctypes.data, est_focal_length, 0, undistort, explicit_camera_centers,
            ctypes.addressof(cams), pts.ctypes.data, use_constraints, use_point_constraints,
            pc.ctypes.data if pc is not None else None, float(point_constraint_weight), int(fix_points), int(optimize_for_fisheye),
            float(eps2),
            ex["V"].ctypes.data if export and "V" in export_keys else None, ex["S"].ctypes.data if export and "S" in export_keys else None,
            ex["U"].ctypes.data if export and "U" in export_keys else None, ex["W"].ctypes.data if export and "W" in export_keys else None]
    info = np.zeros(10)
    if extra_info:
        rc = fn(*args, info.ctypes.data)
    else:
        rc = fn(*args)
    R, c, f, k = cameras_to_arrays(cams)
    return {"rc": rc, "R": R, "c": c, "f": f, "k": k, "pts": pts, "info": info, **ex}


_run_sfm = {}


def run_sfm(scene, optimize_for_fisheye=None, **kw):
    """GPU run_sfm: bsfm_run_sfm, or bsfm_run_sfm_crs for a scene with vis_ptr / vis_cam instead of vmask.  Raises on BSFM
    errors; returns the refined scene + info[10].  Keywords are those of call_run_sfm (known / K_known / k_known for
    calibrated cameras, fisheye / fisheye_params for fisheye cameras).  With optimize_for_fisheye set (0 or 1) the call
    goes to bsfm_run_sfm_fe / bsfm_run_sfm_crs_fe with that value."""
    name = "bsfm_run_sfm_crs" if "vis_ptr" in scene else "bsfm_run_sfm"
    if optimize_for_fisheye is not None:
        name += "_fe"
        kw["optimize_for_fisheye"] = optimize_for_fisheye
    if name not in _run_sfm:
        fn = getattr(load_library(), name)
        _bind_run_sfm(fn)
        if "_crs" in name:   # vmask -> vis_ptr, vis_cam, nvis
            fn.argtypes = fn.argtypes[:3] + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + fn.argtypes[4:]
        fn.argtypes = fn.argtypes + [ctypes.c_void_p]
        fn.restype = ctypes.c_int
        _run_sfm[name] = fn
    out = call_run_sfm(_run_sfm[name], scene, extra_info=True, **kw)
    check(out["rc"], name)
    return out


def last_timing():
    lib = load_library()
    ms = (ctypes.c_float * 6)()
    it, ln = ctypes.c_int(), ctypes.c_int()
    lib.bsfm_ba_last_timing(ms, ctypes.byref(it), ctypes.byref(ln))
    names = ["setup_ms", "jacobian_uvw_ms", "schur_ms", "cholesky_ms", "backsub_eval_ms", "total_ms"]
    d = {k: float(v) for k, v in zip(names, ms)}
    d["iterations"] = it.value
    d["launches"] = ln.value
    return d


def project_known(Pc, K_known, k_known):
    """the calibrated-camera branch of sfm_project_rd (lib/sfm-driver/sfm.c:339-357) on camera-frame points Pc (N x 3)
    with per-point K_known (N x 9) and k_known (N x 5), in the reference's operation order -> pixels (N x 2)"""
    x_n = -Pc[:, 0] / Pc[:, 2]
    y_n = -Pc[:, 1] / Pc[:, 2]
    k, K = k_known, K_known
    rsq = x_n * x_n + y_n * y_n
    factor = 1.0 + k[:, 0] * rsq + k[:, 1] * rsq * rsq + k[:, 4] * rsq * rsq * rsq
    dx_x = 2 * k[:, 2] * x_n * y_n + k[:, 3] * (rsq + 2 * x_n * x_n)
    dx_y = k[:, 2] * (rsq + 2 * y_n * y_n) + 2 * k[:, 3] * x_n * y_n
    x_d = x_n * factor + dx_x
    y_d = y_n * factor + dx_y
    return np.stack([K[:, 0] * x_d + K[:, 1] * y_d + K[:, 2], K[:, 4] * y_d + K[:, 5]], 1)


def reprojection_rmse(scene, sol, known=None, K_known=None, k_known=None):
    """sqrt(mean squared reprojection error) of a solution under the Bundler camera model
    (lib/sfm-driver/sfm.c:302-380), computed in numpy -- a test/bench metric, not a product path.
    known / K_known / k_known: calibrated cameras, as for run_sfm.  Dense or CRS scenes."""
    pi, cj = observations(scene)
    R = sol["R"].reshape(-1, 3, 3)
    Pc = np.einsum("oij,oj->oi", R[cj], sol["pts"][pi] - sol["c"][cj])
    f = sol["f"][cj]
    p = -Pc[:, :2] * f[:, None] / Pc[:, 2:3]
    if known is not None:
        kn = np.asarray(known, bool)[cj]
        if kn.any():
            p[kn] = project_known(Pc[kn], np.asarray(K_known, float).reshape(-1, 9)[cj[kn]], np.asarray(k_known, float)[cj[kn]])
    rsq = (p ** 2).sum(1) / (f * f)
    k = sol["k"][cj]
    p = p * (1.0 + k[:, 0] * rsq + k[:, 1] * rsq * rsq)[:, None]
    e = scene["projections"] - p
    return float(np.sqrt((e ** 2).sum() / e.shape[0]))


def smoke(loader):
    """small BA solve on cuda:0 checked against the oracle (reference build when present)"""
    from . import synth
    scene = synth.ba_scene(10, 500, 4, seed=3)
    got = run_sfm(scene)
    ref = loader.run_sfm_oracle(scene)
    r_gpu, r_ref = np.sqrt(got["info"][1] / scene["projections"].shape[0]), np.sqrt(ref["info"][1] / scene["projections"].shape[0])
    assert abs(r_gpu - r_ref) <= 1e-5, (r_gpu, r_ref)
    assert int(got["info"][5]) == int(ref["info"][5]) and int(got["info"][6]) == int(ref["info"][6])
    print(f"[smoke] BA ok: {int(got['info'][5])} LM iterations, RMSE {r_gpu:.6f} (oracle {r_ref:.6f})")


class SfmModel(ctypes.Structure):
    """== bsfm_sfm_model_t (include/bsfm_b200_ba.h)"""
    _fields_ = [("est_focal_length", ctypes.c_int), ("undistort", ctypes.c_int), ("explicit_camera_centers", ctypes.c_int),
                ("f_scale", ctypes.c_double), ("k_scale", ctypes.c_double),
                ("R_init", ctypes.c_void_p), ("f_fixed", ctypes.c_void_p)]


def pack_params(scene, est_focal_length=1, undistort=1, f_scale=0.001, k_scale=5.0):
    """run_sfm's parameter packing (lib/sfm-driver/sfm.c:652-703) in numpy -> p (m*cnp + 3n doubles)"""
    m, n = len(scene["f"]), scene["pts"].shape[0]
    cnp = 6 + (1 if est_focal_length else 0) + (2 if undistort else 0)
    a = np.zeros((m, cnp))
    a[:, 0:3] = scene["c"]
    c = 6
    if est_focal_length:
        a[:, 6] = scene["f"] * f_scale
        c = 7
    if undistort:
        a[:, c:c + 2] = scene["k"] * k_scale
    return np.concatenate([a.reshape(-1), np.asarray(scene["pts"], float).reshape(-1)]), cnp


def unpack_params(p, scene, est_focal_length=1, undistort=1, f_scale=0.001, k_scale=5.0):
    """run_sfm's unpacking (lib/sfm-driver/sfm.c:876-929) in numpy: p -> dict(R, c, f, k, pts); R = exp([w]x) R_init"""
    m, n = len(scene["f"]), scene["pts"].shape[0]
    cnp = 6 + (1 if est_focal_length else 0) + (2 if undistort else 0)
    a = np.asarray(p[:m * cnp], float).reshape(m, cnp)
    R0 = np.asarray(scene["R"], float).reshape(m, 3, 3)
    R = np.empty_like(R0)
    for j in range(m):
        w = a[j, 3:6]
        th = np.sqrt((w * w).sum())
        if th == 0.0:
            R[j] = R0[j]
            continue
        nx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
        R[j] = (np.eye(3) + nx * np.sin(th) + nx @ nx * (1.0 - np.cos(th))) @ R0[j]
    c = 6
    f = np.asarray(scene["f"], float).copy()
    if est_focal_length:
        f = a[:, 6] / f_scale
        c = 7
    k = a[:, c:c + 2] / k_scale if undistort else np.zeros((m, 2))
    return {"R": R.reshape(m, 9), "c": a[:, 0:3].copy(), "f": f, "k": k, "pts": np.asarray(p[m * cnp:], float).reshape(n, 3).copy()}


def levmar_model(n, m, vmask_ptr, p_ptr, x_ptr, cnp, R_init, f_fixed, est_focal_length=1, undistort=1,
                 explicit_camera_centers=1, eps2=1e-12, itmax=150, verbose=0, jac_mode=0, eps5=4.0e-2, init_params=None,
                 optimize_for_fisheye=None):
    """bsfm_sba_motstr_levmar_model with raw (host or DEVICE) pointers for vmask / p / x.
    init_params: a make_cameras array whose calibrated cameras the projection uses (bsfm_sba_motstr_levmar_model_ki).
    optimize_for_fisheye (0 or 1, with init_params): bsfm_sba_motstr_levmar_model_fe, the fisheye projection with 1.
    Returns (iterations, info[10])."""
    lib = load_library()
    name = "bsfm_sba_motstr_levmar_model" if init_params is None else "bsfm_sba_motstr_levmar_model_ki"
    if optimize_for_fisheye is not None:
        name = "bsfm_sba_motstr_levmar_model_fe"
    fn = getattr(lib, name)
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_void_p,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p] + ([] if init_params is None and optimize_for_fisheye is None else [c.c_void_p]) + \
        ([] if optimize_for_fisheye is None else [c.c_int])
    fn.restype = c.c_int
    R_init = np.ascontiguousarray(R_init, dtype=np.float64)
    f_fixed = np.ascontiguousarray(f_fixed, dtype=np.float64)
    model = SfmModel(est_focal_length, undistort, explicit_camera_centers, 0.001, 5.0, R_init.ctypes.data, f_fixed.ctypes.data)
    opts = np.array([1.0e-3, 1.0e-10, eps2, 1.0e-12, 0.0, eps5])     # sfm.c:705-714 (opts[5] = 4e-2 there)
    info = np.zeros(10)
    args = [n, m, 0, vmask_ptr, p_ptr, cnp, 3, x_ptr, None, 2, ctypes.addressof(model), jac_mode, itmax, verbose,
            opts.ctypes.data, info.ctypes.data, 0, None, 0, None, None, None, None, None]
    if optimize_for_fisheye is not None:
        args += [None if init_params is None else ctypes.addressof(init_params), int(optimize_for_fisheye)]
    elif init_params is not None:
        args.append(ctypes.addressof(init_params))
    rc = fn(*args)
    if rc < -1:
        check(rc, name)
    return rc, info


def mot_levmar_model(n, m, vmask_ptr, p_ptr, x_ptr, points_ptr, cnp, R_init, f_fixed, est_focal_length=1, undistort=1,
                     explicit_camera_centers=1, eps2=1e-12, itmax=150, verbose=0, jac_mode=0, init_params=None,
                     optimize_for_fisheye=None):
    """motion-only counterpart of levmar_model: bsfm_sba_mot_levmar_model(_ki / _fe) with raw (host or DEVICE) pointers for
    vmask / p (cameras only) / x / points (n x 3, fixed).  Returns (iterations, info[10])."""
    lib = load_library()
    name = "bsfm_sba_mot_levmar_model" if init_params is None else "bsfm_sba_mot_levmar_model_ki"
    if optimize_for_fisheye is not None:
        name = "bsfm_sba_mot_levmar_model_fe"
    fn = getattr(lib, name)
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p] + \
        ([] if init_params is None and optimize_for_fisheye is None else [c.c_void_p]) + ([] if optimize_for_fisheye is None else [c.c_int])
    fn.restype = c.c_int
    R_init = np.ascontiguousarray(R_init, dtype=np.float64)
    f_fixed = np.ascontiguousarray(f_fixed, dtype=np.float64)
    model = SfmModel(est_focal_length, undistort, explicit_camera_centers, 0.001, 5.0, R_init.ctypes.data, f_fixed.ctypes.data)
    opts = np.array([1.0e-3, 1.0e-10, eps2, 1.0e-12, 0.0, 4.0e-2])
    info = np.zeros(10)
    args = [n, m, 0, vmask_ptr, p_ptr, cnp, x_ptr, None, 2, ctypes.addressof(model), points_ptr, jac_mode, itmax, verbose,
            opts.ctypes.data, info.ctypes.data, 0, None]
    if optimize_for_fisheye is not None:
        args += [None if init_params is None else ctypes.addressof(init_params), int(optimize_for_fisheye)]
    elif init_params is not None:
        args.append(ctypes.addressof(init_params))
    rc = fn(*args)
    if rc < -1:
        check(rc, name)
    return rc, info


def reprojection_outliers(scene, estimate_distortion=1, min_thresh=8.0, max_thresh=16.0, pt_protected=None, cap=None,
                          known=None, K_known=None, k_known=None, fisheye=None, fisheye_params=None, optimize_for_fisheye=None):
    """bsfm_reprojection_outliers: the statistics / outlier pass BundlerApp::RunSFM_SBA runs after every run_sfm
    (src/Bundle.cpp:659-856) on a scene dict (vmask, projections, R, c, f, k, pts), or bsfm_reprojection_outliers_crs on a
    CRS scene (vis_ptr / vis_cam instead of vmask, see synth.crs_scene).  Defaults are bundler's
    m_min/max_proj_error_threshold (BundlerApp.h).  Returns dist[nvis], stats[m x 5] (n, mean, median, med80, thresh),
    outliers, errors, global_mean.  known / K_known / k_known: calibrated cameras, fisheye / fisheye_params: fisheye
    cameras, as for run_sfm.  With optimize_for_fisheye set (0 or 1) the call goes to the _fe entry with that value."""
    lib = load_library()
    crs = "vis_ptr" in scene
    fe = optimize_for_fisheye is not None
    name = ("bsfm_reprojection_outliers_crs" if crs else "bsfm_reprojection_outliers") + ("_fe" if fe else "")
    fn = getattr(lib, name)
    fn.restype = ctypes.c_int
    vis_types = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] if crs else [ctypes.c_void_p]
    fn.argtypes = [ctypes.c_int, ctypes.c_int] + vis_types + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + \
        ([ctypes.c_int] if fe else []) + [ctypes.c_double, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                   ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    n, m, vis_args, _keep = _visibility_args(scene)
    proj = np.ascontiguousarray(scene["projections"], dtype=np.float64)
    cams = make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], known=known, K_known=K_known, k_known=k_known,
                        fisheye=fisheye, fisheye_params=fisheye_params)
    pts = np.ascontiguousarray(scene["pts"], dtype=np.float64)
    prot = None if pt_protected is None else np.ascontiguousarray(pt_protected, dtype=np.int8)
    nvis = proj.shape[0]
    cap = n if cap is None else int(cap)
    stats = np.zeros((m, 5)); dist = np.zeros(nvis)
    out_idx = np.zeros(max(cap, 1), np.int32); out_err = np.zeros(max(cap, 1))
    gm = ctypes.c_double()
    rc = fn(n, m, *vis_args, proj.ctypes.data, ctypes.addressof(cams), pts.ctypes.data, int(estimate_distortion),
            *([int(optimize_for_fisheye)] if fe else []), float(min_thresh), float(max_thresh), None if prot is None else prot.ctypes.data, stats.ctypes.data, dist.ctypes.data,
            out_idx.ctypes.data, out_err.ctypes.data, cap, ctypes.byref(gm))
    check(rc, name)
    k = min(rc, cap)
    return {"dist": dist, "stats": stats, "outliers": out_idx[:k].copy(), "errors": out_err[:k].copy(), "global_mean": gm.value, "count": rc}


class SfmRound(ctypes.Structure):
    """== bsfm_sfm_round_t (include/bsfm_b200_ba.h)"""
    _fields_ = [("num_pts", ctypes.c_int32), ("nvis", ctypes.c_int32), ("num_outliers", ctypes.c_int32), ("removed", ctypes.c_int32),
                ("info", ctypes.c_double * 10), ("global_mean", ctypes.c_double),
                ("h2d_bytes", ctypes.c_int64), ("h2d_largest", ctypes.c_int64)]


def run_sfm_outlier_loop(scene, est_focal_length=1, undistort=1, explicit_camera_centers=1, ncons=0, eps2=1e-12,
                         use_constraints=0, constrained=None, constraints=None, weights=None,
                         use_point_constraints=0, points_constraints=None, point_constraint_weight=0.0, fix_points=0,
                         known=None, K_known=None, k_known=None, fisheye=None, fisheye_params=None, optimize_for_fisheye=0,
                         remove_outliers=1, min_outliers=40, min_points=20, min_thresh=8.0, max_thresh=16.0, rounds_cap=64,
                         pt_round=True):
    """bsfm_run_sfm_outlier_loop: the solve / outlier-removal loop of BundlerApp::RunSFM_SBA (src/Bundle.cpp:568-919) on a
    CRS scene (synth.crs_scene), with the scene on the GPU between rounds.  Camera and constraint keywords are those of
    call_run_sfm; min_outliers / min_points / min_thresh / max_thresh default to Bundler's.  Returns the refined R, c, f, k,
    pts (by original point index), pt_round, pt_error, cam_stats of the last round, rounds (a list of dicts, at most
    rounds_cap of them), count (rounds run) and mean_error.  pt_round=False passes a null pt_round (refused)."""
    fn = load_library().bsfm_run_sfm_outlier_loop
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_int,
                   c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_double, c.c_int, c.c_int, c.c_double,
                   c.c_int, c.c_int, c.c_int, c.c_double, c.c_double, c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p]
    fn.restype = c.c_int
    assert "vis_ptr" in scene, "run_sfm_outlier_loop takes a CRS scene (synth.crs_scene)"
    n, m, vis_args, _keep = _visibility_args(scene)
    proj = np.ascontiguousarray(scene["projections"], dtype=np.float64)
    cams = make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], constrained, constraints, weights, known, K_known, k_known,
                        fisheye, fisheye_params)
    pts = np.ascontiguousarray(scene["pts"], dtype=np.float64).copy()
    pc = np.ascontiguousarray(points_constraints, dtype=np.float64) if use_point_constraints else None
    rnd = np.full(n, -9, np.int32)
    err = np.zeros(n)
    stats = np.zeros((m, 5))
    rounds = (SfmRound * max(rounds_cap, 1))()
    mean = c.c_double()
    rc = fn(n, m, ncons, *vis_args, proj.ctypes.data, est_focal_length, 0, undistort, explicit_camera_centers,
            c.addressof(cams), pts.ctypes.data, use_constraints, use_point_constraints, pc.ctypes.data if pc is not None else None,
            float(point_constraint_weight), int(fix_points), int(optimize_for_fisheye), float(eps2),
            int(remove_outliers), int(min_outliers), int(min_points), float(min_thresh), float(max_thresh),
            rnd.ctypes.data if pt_round else None, err.ctypes.data, stats.ctypes.data, c.addressof(rounds), int(rounds_cap), c.byref(mean))
    check(rc, "bsfm_run_sfm_outlier_loop")
    R, cc, f, k = cameras_to_arrays(cams)
    out_rounds = [{"num_pts": r.num_pts, "nvis": r.nvis, "num_outliers": r.num_outliers, "removed": r.removed,
                   "info": np.array(list(r.info)), "global_mean": r.global_mean, "h2d_bytes": r.h2d_bytes, "h2d_largest": r.h2d_largest}
                  for r in rounds[:min(rc, rounds_cap)]]
    return {"count": rc, "R": R, "c": cc, "f": f, "k": k, "pts": pts, "pt_round": rnd, "pt_error": err, "cam_stats": stats,
            "rounds": out_rounds, "mean_error": mean.value}
