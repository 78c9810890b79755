"""numpy restatements of the reference's fisheye projections, shared by the golden-file generator and the tests.

  - port_run_sfm_fisheye: run_sfm with optimize_for_fisheye = 1 (motion + structure): tests/ba_restatement.py's LM
    restatement with its projection replaced by sfm_project_point2_fisheye (lib/sfm-driver/sfm.c:448-492), i.e. the
    pinhole of sfm_project2 (:243-299) without the radial step, then sfm_fisheye_distort (:426-446).
  - reprojection_outliers_fisheye: the outlier pass of BundlerApp::RunSFM_SBA with m_optimize_for_fisheye
    (src/Bundle.cpp:659-856): sfm_project_rd (the unmodified reference function when oracle/_ref is built, else
    oracle/outlier_oracle.py's port), then ImageData::DistortPoint (ImageData.cpp:1129-1169) restated here with
    GetRotationFromSpherical (BundleUtil.cpp:70-94), then the statistics of oracle/outlier_oracle.py."""
import ctypes
import math
from unittest import mock

import numpy as np

from bundler_sfm_b200 import bundle, synth
from oracle import outlier_oracle
from tests import ba_restatement as BR


def project_rows_fisheye(P, fisheye, fisheye_params, a, b, R):
    """sfm_project_point2_fisheye for the observation rows a / b / R of a ba_restatement problem"""
    cj = P.cj
    u = BR.project_rows(a, b, R, P.f_fixed[cj], P.kn[cj], P.Kk[cj], P.kk[cj], P.est_focal, 0, P.explicit_centers)
    fe = np.asarray(fisheye)[cj] != 0
    if fe.any():
        u[fe] = synth.fisheye_map(u[fe], np.asarray(fisheye_params, float)[cj[fe]])
    return u


def port_run_sfm_fisheye(scene, fisheye, fisheye_params, **kw):
    """ba_restatement.port_run_sfm (keywords as bundle.call_run_sfm) with the fisheye projection in every residual and
    forward-difference evaluation"""
    def evaluate(P, pp, a=None, b=None, R=None):
        A_ = pp[:P.ncp].reshape(P.m, P.cnp)[P.cj] if a is None else a
        B_ = pp[P.ncp:].reshape(P.n, 3)[P.pi] if b is None else b
        R_ = BR.rot_update_rows(P.R_init[P.cj], A_[:, 3:6]) if R is None else R
        return project_rows_fisheye(P, fisheye, fisheye_params, A_, B_, R_)
    with mock.patch.object(BR, "evaluate", evaluate):
        return BR.port_run_sfm(scene, **kw)


def rotation_from_spherical(theta, phi):
    """GetRotationFromSpherical (src/BundleUtil.cpp:70-94) with the C library's cos / sin -> R (9, row-major)"""
    v = [math.cos(theta) * math.sin(phi), math.cos(phi), math.sin(theta) * math.sin(phi)]
    phi_up, theta_up = phi - 0.5 * math.pi, theta
    up = [math.cos(theta_up) * math.sin(phi_up), math.cos(phi_up), math.sin(theta_up) * math.sin(phi_up)]
    x_axis = [v[1] * up[2] - v[2] * up[1], v[2] * up[0] - v[0] * up[2], v[0] * up[1] - v[1] * up[0]]   # matrix_cross
    return x_axis + up + v


R_DISTORT = rotation_from_spherical(-0.5 * math.pi, 0.5 * math.pi)     # ImageData::DistortPoint(x, y, x_out, y_out)


def distort_point(x, y, fp, R=R_DISTORT):
    """ImageData::DistortPoint (ImageData.cpp:1138-1169) of a fisheye camera with fp = (f_cx, f_cy, f_rad, f_angle,
    f_focal); a ray whose rotated z is <= 0 leaves (x, y) as it is (the reference returns without writing)"""
    cx, cy, rad, fang, F = (float(v) for v in fp)
    ray = (x, y, -F)
    rot = [R[3 * r] * ray[0] + R[3 * r + 1] * ray[1] + R[3 * r + 2] * ray[2] for r in range(3)]
    if rot[2] <= 0.0:
        return x, y
    xn = rot[0] * F / rot[2]
    yn = rot[1] * F / rot[2]
    r = math.sqrt(xn * xn + yn * yn)
    angle = math.atan(r / F) * (180.0 / math.pi)                     # RAD2DEG, imagelib/defines.h:32
    rnew = rad * angle / (0.5 * fang)
    return xn * (rnew / r) + cx, yn * (rnew / r) + cy


def reprojection_outliers_fisheye(scene, estimate_distortion=1, min_thresh=8.0, max_thresh=16.0, pt_protected=None,
                                  optimize_for_fisheye=1, use_reference=True):
    """the outlier pass (src/Bundle.cpp:659-856) on ordinary / fisheye cameras (scene: vmask, projections, R, c, f, k, pts,
    fisheye, fisheye_params).  Returns the dict of outlier_oracle.reprojection_outliers."""
    lib = None
    if use_reference:
        from oracle import loader
        lib = loader.ref_sba()
    vm = np.asarray(scene["vmask"]) != 0
    n, m = vm.shape
    obs_pt, obs_cam = np.nonzero(vm)
    proj = np.asarray(scene["projections"], float)
    pts = np.ascontiguousarray(scene["pts"], float)
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], fisheye=scene["fisheye"],
                               fisheye_params=scene["fisheye_params"])
    if lib is not None:
        fn = lib.sfm_project_rd
        fn.restype = ctypes.c_int
        fn.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int, ctypes.c_int]
        kth = lib.kth_element_copy
        kth.restype = ctypes.c_double
        kth.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    size = ctypes.sizeof(bundle.CameraParams)
    base = ctypes.addressof(cams)
    dist = np.zeros(len(obs_pt))
    for o, (i, j) in enumerate(zip(obs_pt, obs_cam)):
        i, j = int(i), int(j)
        if lib is not None:
            cam = bundle.CameraParams.from_address(base + j * size)
            K = (ctypes.c_double * 9)(cam.f, 0, 0, 0, cam.f, 0, 0, 0, 1)                        # Bundle.cpp:670-672
            dt = (ctypes.c_double * 3)(cam.t[0], cam.t[1], cam.t[2])
            b = (ctypes.c_double * 3)(*pts[i])
            pr = (ctypes.c_double * 2)()
            fn(base + j * size, K, ctypes.addressof(cam) + bundle.CameraParams.k.offset, ctypes.addressof(cam), dt, b, pr,
               int(estimate_distortion), 1)
            p0, p1 = pr[0], pr[1]
        else:
            p0, p1 = outlier_oracle._project_port(np.asarray(scene["R"][j]).reshape(-1), scene["c"][j], float(scene["f"][j]),
                                                  scene["k"][j], pts[i], estimate_distortion)
        if optimize_for_fisheye and scene["fisheye"][j]:                                       # Bundle.cpp:746-751
            p0, p1 = distort_point(float(p0), float(p1), scene["fisheye_params"][j])
        dx, dy = p0 - proj[o, 0], p1 - proj[o, 1]
        dist[o] = math.sqrt(dx * dx + dy * dy)
    stats = np.zeros((m, 5))
    outliers, errors, first_cam = [], [], []
    tot, cnt = 0.0, 0
    for j in range(m):
        sel = np.nonzero(obs_cam == j)[0]
        d = np.ascontiguousarray(dist[sel])
        nj = len(d)
        k80, k50 = outlier_oracle.iround(0.8 * nj), outlier_oracle.iround(0.5 * nj)
        if lib is not None and nj > 0:
            med80 = kth(nj, k80, d.ctypes.data) if k80 < nj else 0.0
            med50 = kth(nj, k50, d.ctypes.data) if k50 < nj else 0.0
        else:
            med80, med50 = outlier_oracle._kth_port(d, k80), outlier_oracle._kth_port(d, k50)
        thresh = 1.2 * 2.0 * med80
        thresh = min_thresh if thresh < min_thresh else (max_thresh if thresh > max_thresh else thresh)
        s = 0.0
        for v in d:
            s += v
        stats[j] = (nj, s / nj if nj else np.nan, med50, med80, thresh)
        tot += s; cnt += nj
        for q, o in enumerate(sel):
            i = int(obs_pt[o])
            if pt_protected is not None and pt_protected[i]:
                continue
            if d[q] > thresh and i not in outliers:
                outliers.append(i); errors.append(float(d[q])); first_cam.append(j)
    order = sorted(range(len(outliers)), key=lambda q: (first_cam[q], outliers[q]))
    return {"dist": dist, "stats": stats, "outliers": np.array([outliers[q] for q in order], dtype=np.int32),
            "errors": np.array([errors[q] for q in order]), "global_mean": tot / cnt}
