"""The BA linear algebra kernel by kernel, at chosen points, against the numpy restatement in tests/ba_restatement.py.

The end-to-end BA tests compare whole solves, and LM hides a lot: the gradient J^T e is exact and a step only has to go
downhill.  These tests compare one kernel's output entry by entry instead.

- Normal-equation blocks (bsfm_sba_motstr_levmar_model with itmax = 0): the export pass forms U, V, W and the undamped
  S = blockdiag(U) - W V^-1 W^T from one Jacobian at the p the test passes in.
  - S is recomputed in long double from the GPU's own exported U, V and W.  That isolates schur_partial_kernel /
    schur_final_kernel from the Jacobian.  The gate is the summation error bound, not a tuned constant.
  - In analytic mode (jacobian_kernel, jac_mode = 1), U / V / W are compared with the exact Jacobian (complex-step).
  - In FD mode (jac_mode = 0), U / V / W are compared with the numpy forward differences.  The gate is their rounding
    bound, propagated to the blocks.
- Scenes are built from a camera graph, so that the Schur blocks have chosen tuple counts: 1 to 5 chunks of 64 tuples,
  rings shorter and longer than the 8-deep cp.async ring, camera pairs without a common point, a complete graph, U
  accumulated in 2 segments, and a lopsided scene with 32 segments, many of them empty.
- One LM iteration (itmax = 1, first trial step accepted) is compared with the restatement's damped step (analytic mode),
  and with the unmodified reference run for one iteration (FD mode), at mcon 0 and 2, with constraints, in every cnp and in
  each dense-Cholesky regime.  The motion-only step is compared in the same way."""
import ctypes
import os

import numpy as np
import pytest

from bundler_sfm_b200 import bundle, synth
from tests import ba_restatement as rs

u = rs.U_ROUND
MODES = [(0, 0), (1, 0), (0, 1), (1, 1)]          # (est_focal_length, undistort): cnp = 6, 7, 8, 9


# ---- scenes ---------------------------------------------------------------------------------------------------------
def graph_scene(m, pairs=(), groups=(), seed=0, explicit_centers=1, focal=800.0, pixel_noise=0.5):
    """cameras on a ring looking at the unit cube; `pairs` = [(j, k, count)]: count points seen by exactly cameras j and k;
    `groups` = [(cameras, count)]: count points seen by exactly those cameras.  Every point has at least two views, so every
    V_i is invertible.  Measurements come from the true cameras with radial distortion, plus noise; the initial estimate is
    perturbed.  With explicit_centers = 0 the translation t = -R c is stored in "c", which is what run_sfm then reads."""
    rng = np.random.default_rng(seed)
    views = [(j, k) for j, k, cnt in pairs for _ in range(cnt)] + [tuple(cams) for cams, cnt in groups for _ in range(cnt)]
    n = len(views)
    ang = 2.0 * np.pi * np.arange(m) / m
    c = np.stack([6.0 * np.cos(ang), 0.3 * np.sin(3 * ang), 6.0 * np.sin(ang)], 1)
    R = np.zeros((m, 3, 3))
    for j in range(m):
        z = c[j] / np.linalg.norm(c[j])
        xax = np.cross(np.array([0.0, 1.0, 0.0]), z); xax /= np.linalg.norm(xax)
        R[j] = np.stack([xax, np.cross(z, xax), z], 0)
    vmask = np.zeros((n, m), np.int8)
    for i, cams in enumerate(views):
        vmask[i, list(cams)] = 1
    pts = rng.uniform(-1.0, 1.0, (n, 3))
    k_true = np.stack([rng.uniform(-0.08, -0.02, m), rng.uniform(0.005, 0.02, m)], 1)
    pi, cj = np.nonzero(vmask)
    Pc = np.einsum("oij,oj->oi", R[cj], pts[pi] - c[cj])
    proj = -Pc[:, :2] * focal / Pc[:, 2:3]
    rsq = (proj ** 2).sum(1) / focal ** 2
    proj *= (1.0 + k_true[cj, 0] * rsq + k_true[cj, 1] * rsq * rsq)[:, None]
    proj += pixel_noise * rng.standard_normal(proj.shape)
    c0 = c + 0.01 * rng.standard_normal(c.shape)
    return {"vmask": vmask, "projections": np.ascontiguousarray(proj), "R": R.reshape(m, 9).copy(),
            "c": c0 if explicit_centers else -np.einsum("jab,jb->ja", R, c0),
            "f": focal * (1.0 + 0.01 * rng.standard_normal(m)), "k": k_true + 0.003 * rng.standard_normal((m, 2)),
            "pts": pts + 0.02 * rng.standard_normal(pts.shape), "gt_pts": pts}


def _chunks_scene(ec):
    # off-diagonal Schur blocks of 1, 7, 8, 9, 63, 64, 65, 256 and 257 tuples (1 to 5 chunks of 64; rings shorter and longer
    # than 8; 5 chunks = one group of four + a partial group), and most camera pairs without a common point
    pairs = [(0, 1, 1), (0, 2, 7), (1, 3, 8), (2, 4, 9), (3, 5, 63), (4, 6, 64), (5, 7, 65), (6, 8, 256), (7, 9, 257), (8, 9, 2),
             (1, 2, 3)]
    return graph_scene(10, pairs, seed=1, explicit_centers=ec)


def _complete_scene(ec):
    # every camera pair shares points; points with 2 to 6 views
    pairs = [(j, k, 2 + (3 * j + k) % 5) for j in range(6) for k in range(j + 1, 6)]
    return graph_scene(6, pairs, groups=[((0, 1, 2), 11), ((1, 3, 4, 5), 9), (tuple(range(6)), 20)], seed=2, explicit_centers=ec)


def _useg2_scene(ec):
    # ~2000 observations per camera: U is accumulated in 2 segments per camera
    return graph_scene(3, groups=[((0, 1, 2), 2000)], seed=3, explicit_centers=ec)


def _lopsided_scene(ec):
    # 127 k observations on 4 cameras: 32 segments per camera, but cameras 2 and 3 have 8 and 7 observations, so most of
    # their segments are empty
    return graph_scene(4, [(0, 1, 63600), (2, 3, 5), (0, 2, 3), (1, 3, 2)], seed=4, explicit_centers=ec)


SCENES = {"chunks": _chunks_scene, "complete": _complete_scene, "useg2": _useg2_scene, "lopsided": _lopsided_scene}


def useg_of(scene):                # ba_solver.cu: observations per U-accumulation CTA
    nvis, m = int(np.count_nonzero(scene["vmask"])), scene["vmask"].shape[1]
    return max(1, min(32, (nvis // m + 1023) // 1024))


def constraints_for(scene, cnp, seed=0):
    """camera constraints on every third camera (three parameters each) and point constraints on every fifth point, in
    run_sfm's keyword form"""
    m = len(scene["f"])
    rng = np.random.default_rng(seed)
    constrained = np.zeros((m, 9), np.int8); cons = np.zeros((m, 9)); wts = np.zeros((m, 9))
    for j in range(0, m, 3):
        for q in (0, 4, cnp - 1):
            constrained[j, q] = 1
            wts[j, q] = rng.uniform(0.5, 2.0) * (1e-6 if (cnp >= 7 and q == 6) else 1.0)    # weights in run_sfm's units
    cons[:, 0:3] = scene["c"] + 0.005
    cons[:, 6] = scene["f"] * 1.002
    pc = np.zeros_like(scene["pts"])
    pc[::5] = scene["gt_pts"][::5]
    return dict(use_constraints=1, constrained=constrained, constraints=cons, weights=wts,
                use_point_constraints=1, points_constraints=pc, point_constraint_weight=0.3)


def with_rotation_increments(P, p):
    """nonzero w on cameras 1 and 2: theta^2 = 1.4e-9 (< 1e-8, the series branch of (1 - cos)/theta^2 in the analytic
    Jacobian) and 7.25e-6 (the closed form); camera 0 keeps w = 0"""
    p = p.copy()
    a = p[:P.ncp].reshape(P.m, P.cnp)
    a[1, 3:6] = (2e-5, -1e-5, 3e-5)
    a[2, 3:6] = (1e-3, 2e-3, -1.5e-3)
    return p


# ---- the C entry points ---------------------------------------------------------------------------------------------
class CamCons(ctypes.Structure):          # == bsfm_camera_constraints_t
    _fields_ = [("constrained", ctypes.c_void_p), ("constraints", ctypes.c_void_p), ("weights", ctypes.c_void_p)]


class PtCons(ctypes.Structure):           # == bsfm_point_constraints_t
    _fields_ = [("constrained", ctypes.c_char), ("constraints", ctypes.c_double * 3), ("weight", ctypes.c_double)]


OPTS = np.array([1.0e-3, 1.0e-10, 1e-12, 1.0e-12, 0.0, 4.0e-2])      # sfm.c:705-714


def _constraint_args(P):
    keep = []
    cam = None
    if P.use_constraints:
        cc = np.ascontiguousarray(P.cc, np.int8); cv = np.ascontiguousarray(P.cv); cw = np.ascontiguousarray(P.cw)
        keep += [cc, cv, cw]
        cam = (CamCons * P.m)()
        for j in range(P.m):
            cam[j].constrained = cc.ctypes.data + j * P.cnp
            cam[j].constraints = cv.ctypes.data + 8 * j * P.cnp
            cam[j].weights = cw.ctypes.data + 8 * j * P.cnp
    pt = None
    if P.use_point_constraints:
        pt = (PtCons * P.n)()
        for i in np.nonzero(P.pc)[0]:
            pt[i].constrained = b"\x01"
            pt[i].constraints[:] = list(P.pv[i])
            pt[i].weight = P.pw
    return cam, pt, keep


def gpu_motstr(P, p, jac_mode, itmax, export=False, eps5=OPTS[5]):
    """bsfm_sba_motstr_levmar_model on the problem P from p (host pointers) -> (rc, p_out, info, blocks); eps5 = 0 disables
    the stop-8 rule"""
    lib = bundle.load_library()
    fn = lib.bsfm_sba_motstr_levmar_model
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_void_p,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p]
    fn.restype = c.c_int
    R_init = np.ascontiguousarray(P.R_init); f_fixed = np.ascontiguousarray(P.f_fixed)
    model = bundle.SfmModel(P.est_focal, P.undistort, P.explicit_centers, rs.F_SCALE, rs.K_SCALE, R_init.ctypes.data, f_fixed.ctypes.data)
    vm = np.ascontiguousarray(P.vm, np.int8); x = np.ascontiguousarray(P.x).reshape(-1).copy()
    pp = np.ascontiguousarray(p, np.float64).copy()
    cam, pt, keep = _constraint_args(P)
    opts = OPTS.copy()
    opts[5] = eps5
    info = np.zeros(10)
    ex = {}
    if export:
        ex = {"V": np.zeros((P.n, 9)), "S": np.zeros((P.ncp, P.ncp)), "U": np.zeros((P.m, P.cnp * P.cnp)),
              "W": np.zeros((P.ncp, 3 * P.n))}
    rc = fn(P.n, P.m, P.mcon, vm.ctypes.data, pp.ctypes.data, P.cnp, 3, x.ctypes.data, None, 2, ctypes.addressof(model),
            jac_mode, itmax, 0, opts.ctypes.data, info.ctypes.data,
            P.use_constraints, ctypes.addressof(cam) if cam is not None else None,
            P.use_point_constraints, ctypes.addressof(pt) if pt is not None else None,
            *[ex[k].ctypes.data if export else None for k in ("V", "S", "U", "W")])
    blocks = None
    if export:
        W = ex["W"].reshape(P.m, P.cnp, P.n, 3)[P.cj, :, P.pi, :]          # per observation, cnp x 3
        blocks = dict(U=ex["U"].reshape(P.m, P.cnp, P.cnp), V=ex["V"].reshape(P.n, 3, 3), W=W, S=ex["S"])
    return rc, pp, info, blocks


def gpu_mot(P, p_cams, jac_mode, itmax):
    """bsfm_sba_mot_levmar_model (points fixed at P.p0's) -> (rc, cameras out, info)"""
    lib = bundle.load_library()
    fn = lib.bsfm_sba_mot_levmar_model
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p]
    fn.restype = c.c_int
    R_init = np.ascontiguousarray(P.R_init); f_fixed = np.ascontiguousarray(P.f_fixed)
    model = bundle.SfmModel(P.est_focal, P.undistort, P.explicit_centers, rs.F_SCALE, rs.K_SCALE, R_init.ctypes.data, f_fixed.ctypes.data)
    vm = np.ascontiguousarray(P.vm, np.int8); x = np.ascontiguousarray(P.x).reshape(-1).copy()
    a = np.ascontiguousarray(p_cams, np.float64).copy()
    pts = np.ascontiguousarray(P.p0[P.ncp:]).copy()
    cam, _, keep = _constraint_args(P)
    info = np.zeros(10)
    rc = fn(P.n, P.m, P.mcon, vm.ctypes.data, a.ctypes.data, P.cnp, x.ctypes.data, None, 2, ctypes.addressof(model),
            pts.ctypes.data, jac_mode, itmax, 0, OPTS.ctypes.data, info.ctypes.data,
            P.use_constraints, ctypes.addressof(cam) if cam is not None else None)
    return rc, a, info


# ---- reference values and bounds in numpy ---------------------------------------------------------------------------
def schur_longdouble(P, U, V, W):
    """diag(U) - sum_i W_i V_i^-1 W_i^T in long double from the given blocks, and the summation bound of an fp64
    evaluation: c u (|U| + sum_i kappa(V_i) |W_ij| |V_i^-1| |W_ik|^T) per entry, c = (tuples per chunk) + (chunks) + 12"""
    ld = np.longdouble
    m, n, cnp = P.m, P.n, P.cnp
    Vl = V.astype(ld)
    Vinv = np.linalg.inv(V)                       # fp64, for the bound only
    kap = np.linalg.cond(V)
    # exact-ish inverse in long double: one Newton step on the fp64 inverse, X (2I - V X)
    Xl = Vinv.astype(ld)
    I3 = np.eye(3, dtype=ld)[None]
    Xl = np.einsum("nab,nbc->nac", Xl, 2 * I3 - np.einsum("nab,nbc->nac", Vl, Xl))
    S = np.zeros((m * cnp, m * cnp), ld)
    T = np.zeros((m * cnp, m * cnp))
    ntup = np.zeros((m, m), int)
    for j in range(m):
        S[j * cnp:(j + 1) * cnp, j * cnp:(j + 1) * cnp] = U[j].astype(ld)
        T[j * cnp:(j + 1) * cnp, j * cnp:(j + 1) * cnp] = np.abs(U[j])
    Wl = W.astype(ld)
    Y = np.einsum("oab,obc->oac", Wl, Xl[P.pi])
    Ya = np.einsum("oab,obc->oac", np.abs(W), np.abs(Vinv[P.pi])) * kap[P.pi][:, None, None]
    start = np.searchsorted(P.pi, np.arange(n + 1))
    counts = np.diff(start)
    for L in np.unique(counts):
        pts = np.nonzero(counts == L)[0]
        for s in range(L):
            for t in range(L):
                o1, o2 = start[pts] + s, start[pts] + t
                j, k = P.cj[o1], P.cj[o2]
                blk = np.einsum("oab,ocb->oac", Y[o1], Wl[o2])
                blkT = np.einsum("oab,ocb->oac", Ya[o1], np.abs(W[o2]))
                rows = (j * cnp)[:, None, None] + np.arange(cnp)[None, :, None]
                cols = (k * cnp)[:, None, None] + np.arange(cnp)[None, None, :]
                np.subtract.at(S, (rows, cols), blk)
                np.add.at(T, (rows, cols), blkT)
                np.add.at(ntup, (j, k), 1)
    cblk = np.minimum(ntup, 64) + (ntup + 63) // 64 + 12
    c = np.repeat(np.repeat(cblk, cnp, 0), cnp, 1)
    return S, c * u * T


def fd_block_bound(P, A, B, eA, eB, c_fd=32.0):
    """per-entry bound on |U_gpu - U_np|, |V_gpu - V_np|, |W_gpu - W_np| when both sides form forward differences: each
    Jacobian entry is off by at most c_fd eA (both evaluations of h, on both sides), and the sums by (count + 4) u sum|terms|"""
    dA, dB = c_fd * eA, c_fd * eB
    aA, aB = np.abs(A), np.abs(B)
    sel, cj, pi = P.sel, P.cj, P.pi
    cnt_c = np.bincount(cj, minlength=P.m) + 4.0
    cnt_p = np.bincount(pi, minlength=P.n) + 4.0
    bU = np.zeros((P.m, P.cnp, P.cnp))
    np.add.at(bU, cj[sel], np.einsum("oki,okj->oij", dA[sel], aA[sel]) + np.einsum("oki,okj->oij", aA[sel], dA[sel])
              + u * cnt_c[cj[sel], None, None] * np.einsum("oki,okj->oij", aA[sel], aA[sel]))
    bV = np.zeros((P.n, 3, 3))
    np.add.at(bV, pi, np.einsum("oki,okj->oij", dB, aB) + np.einsum("oki,okj->oij", aB, dB)
              + u * cnt_p[pi, None, None] * np.einsum("oki,okj->oij", aB, aB))
    bW = np.einsum("oki,okj->oij", dA, aB) + np.einsum("oki,okj->oij", aA, dB) + 4 * u * np.einsum("oki,okj->oij", aA, aB)
    return bU, bV, bW


def _case(name, ef, ud, ec, jac_mode):
    """the blocks the GPU exports at p0 + rotation increments, with camera and point constraints"""
    scene = SCENES[name](ec)
    cnp = 6 + ef + 2 * ud
    kw = dict(est_focal_length=ef, undistort=ud, explicit_camera_centers=ec, **constraints_for(scene, cnp))
    P = rs.problem(scene, **kw)
    p = with_rotation_increments(P, P.p0)
    rc, _, _, blocks = gpu_motstr(P, p, jac_mode, 0, export=True)
    assert rc == 0, (name, rc, bundle.load_library().bsfm_last_error())
    return P, p, blocks


BLOCK_CASES = [(name, ef, ud, ec) for name in SCENES for ef, ud in MODES for ec in (1, 0)]


def _ids(c):
    return f"{c[0]}-ef{c[1]}ud{c[2]}-ec{c[3]}"


# ---- CPU: the scenes have the shapes they are meant to have ---------------------------------------------------------
def test_scene_shapes():
    sc = _chunks_scene(1)
    P = rs.problem(sc)
    ntup = np.zeros((P.m, P.m), int)
    for i in range(P.n):
        cams = P.cj[P.pi == i]
        for a in cams:
            for b in cams:
                ntup[a, b] += a < b
    assert sorted(ntup[ntup > 0].tolist()) == [1, 2, 3, 7, 8, 9, 63, 64, 65, 256, 257]
    assert (ntup + ntup.T == 0).sum() > P.m * P.m // 2                  # camera pairs without a common point
    cp = rs.problem(_complete_scene(1))
    assert all(cp.vm[:, j].astype(int) @ cp.vm[:, k].astype(int) > 0 for j in range(6) for k in range(6))
    assert useg_of(_useg2_scene(1)) == 2
    lop = _lopsided_scene(1)
    assert useg_of(lop) == 32
    per_cam = lop["vmask"].sum(0)
    assert per_cam.min() < 32 < per_cam.max()                            # cameras with empty segments
    for name, make in SCENES.items():
        assert make(1)["vmask"].sum(1).min() >= 2, name


def test_complex_step_matches_central_differences():
    """the exact Jacobian (complex-step through the restated rotation update and projection) against central differences,
    at rotation increments 0, 3e-5 and 2.7e-3, with explicit centres on and off: agreement at the central differences'
    truncation error"""
    for ec in (1, 0):
        sc = _complete_scene(ec)
        P = rs.problem(sc, explicit_camera_centers=ec)
        p = with_rotation_increments(P, P.p0)
        A, B = rs.jacobian_exact(P, p)
        a, b, _ = rs._obs_rows(P, p)
        for jj in range(P.cnp):
            h = 1e-6 * max(1.0, float(np.max(np.abs(a[:, jj]))))
            ap, am = a.copy(), a.copy(); ap[:, jj] += h; am[:, jj] -= h
            cd = (rs.evaluate(P, p, ap, b) - rs.evaluate(P, p, am, b)) / (2 * h)
            assert np.max(np.abs(cd - A[:, :, jj])) <= 1e-6 * np.max(np.abs(A[:, :, jj])), (ec, jj)
        for jj in range(3):
            bp, bm = b.copy(), b.copy(); bp[:, jj] += 1e-6; bm[:, jj] -= 1e-6
            cd = (rs.evaluate(P, p, a, bp) - rs.evaluate(P, p, a, bm)) / 2e-6
            assert np.max(np.abs(cd - B[:, :, jj])) <= 1e-6 * np.max(np.abs(B[:, :, jj])), (ec, jj)


# ---- CPU: the restatement against the unmodified reference -----------------------------------------------------------
def _ref_or_skip():
    from oracle import loader
    if loader.ref_sba() is None:
        pytest.skip("needs oracle/_ref (the unmodified reference build)")
    return loader


def _ref_run(loader, scene, itmax, monkeypatch, **kw):
    monkeypatch.setenv("REF_SBA_ITMAX", str(itmax))
    return loader.run_sfm_ref(scene, **kw)


# The blocks are pinned to the reference only indirectly, through test_one_fd_iteration_restatement_vs_reference below.  The
# reference's own Uout / Vout / Wout / Sout cannot serve: with itmax = 0 it verifies its Jacobian and returns before the
# export (sba_levmar.c:769), and its export pass segfaults inside the reference on every scene with two-view points tried
# here (these graph scenes, and synth.ba_scene(6, 120, 2)); scenes whose points all have three or more views export fine.
#
# One FD iteration, restatement against the reference, measured per case: the largest relative difference per parameter
# group (max |diff| over the group's max |value|) and the largest relative difference of info[1..4].  The GPU is gated at
# ten times the case's own spread.
FD_SPREAD = {                       # case: (parameters, info)
    "small-cnp9-cons": (4.23e-13, 7.50e-12),
    "small-cnp6-tcam-mcon2": (1.01e-12, 8.42e-14),
    "small-cnp8-mcon2-cons": (4.07e-13, 2.83e-12),
    "fused-cnp7": (1.30e-12, 3.06e-12),
    "tile-cnp9-mcon2-cons": (2.56e-11, 5.09e-12),
}


def rel_group_err(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _step_spread(got, ref):
    return max(rel_group_err(got[k], ref[k]) for k in ("R", "c", "f", "k", "pts"))


def _info_spread(got, ref):
    return max(abs(got["info"][q] - ref["info"][q]) / abs(ref["info"][q]) for q in (1, 2, 3, 4))


# (scene maker, est_focal_length, undistort, explicit centres, mcon, constraints): every cnp, mcon 0 and 2, camera and point
# constraints, reduced systems of 36..1350 unknowns: the dataflow path (<= 640), the fused steps (641..1248) and the tile
# kernel (1249..1536)
def _small(ec):
    return _complete_scene(ec)


def _fused(ec):                     # cnp 7: 100 cameras -> 700 unknowns
    return synth.ba_scene(100, 2500, 4, seed=61)


def _tile(ec):                      # cnp 9: 150 cameras, 2 fixed -> 1332 unknowns
    return synth.ba_scene(150, 3000, 4, seed=62)


STEP_CASES = {
    "small-cnp9-cons": (_small, 1, 1, 1, 0, True),
    "small-cnp6-tcam-mcon2": (_small, 0, 0, 0, 2, False),
    "small-cnp8-mcon2-cons": (_small, 0, 1, 1, 2, True),
    "fused-cnp7": (_fused, 1, 0, 1, 0, False),
    "tile-cnp9-mcon2-cons": (_tile, 1, 1, 1, 2, True),
}


def _step_problem(name):
    make, ef, ud, ec, mcon, cons = STEP_CASES[name]
    sc = make(ec)
    if "gt_pts" not in sc:
        sc["gt_pts"] = sc["pts"]
    cnp = 6 + ef + 2 * ud
    kw = dict(est_focal_length=ef, undistort=ud, explicit_camera_centers=ec, ncons=mcon)
    if cons:
        kw.update(constraints_for(sc, cnp, seed=5))
    return sc, kw


@pytest.mark.parametrize("name", list(STEP_CASES))
def test_one_fd_iteration_restatement_vs_reference(name, monkeypatch):
    """the restatement's FD iteration against the reference's, at the same point: this is the spread the GPU gate is built on"""
    loader = _ref_or_skip()
    sc, kw = _step_problem(name)
    ref = _ref_run(loader, sc, 1, monkeypatch, **kw)
    got = rs.port_run_sfm(sc, itmax=1, **kw)
    # the reference counts the Jacobian's function evaluations in nfev (info[7]); one linear system on both sides
    assert int(got["info"][7]) == 2 and int(ref["info"][9]) == int(got["info"][9]) == 1 and int(ref["info"][5]) == 1
    assert _step_spread(got, ref) <= 2 * FD_SPREAD[name][0], _step_spread(got, ref)
    assert _info_spread(got, ref) <= 2 * FD_SPREAD[name][1], _info_spread(got, ref)


# ---- GPU: normal-equation blocks ---------------------------------------------------------------------------------------
# Every check below is a ratio error / bound; a test passes when every ratio is <= 1.  The *_ratios functions return them
# so that the margins can be listed.
def schur_ratios(case):
    """schur_partial_kernel / schur_final_kernel: the exported undamped S against diag(U) - sum W V^-1 W^T in long double
    from the GPU's own U, V and W, over the summation bound of schur_longdouble"""
    P, p, g = _case(*case, 0)
    S, bound = schur_longdouble(P, g["U"], g["V"], g["W"])
    err = np.abs(g["S"].astype(np.longdouble) - S).astype(float)
    return {"S": float(np.max(err / np.maximum(bound, 1e-300)))}


# Analytic blocks against the exact Jacobian, each entry scaled by its two column norms.  The analytic kernel and the
# complex-step restatement round differently inside the chain rule (rotation columns through -[Pc]x J_l(w), the distortion
# and the perspective division), and one block entry sums up to 2k observations; the largest scaled difference measured on
# an H100 over all BLOCK_CASES was 1.8e-12 (U of the chunks scene, ec = 1; V 1.4e-15, W 9.1e-13).  ANALYTIC_GATE is about
# five times that.  A wrong column, a lost term or a missing segment gives >= 1e-3.
ANALYTIC_GATE = 1e-11


def analytic_ratios(case):
    """jacobian_kernel<false> (jac_mode = 1) + u_partial / u_final / v_kernel against U / V / W of the complex-step
    Jacobian"""
    P, p, g = _case(*case, 1)
    A, B = rs.jacobian_exact(P, p)
    blk = rs.normal_blocks(P, p, A, B, P.x - rs.evaluate(P, p))
    du = np.sqrt(np.diagonal(blk.U, axis1=1, axis2=2))
    dv = np.sqrt(np.diagonal(blk.V, axis1=1, axis2=2))
    eu = np.abs(g["U"] - blk.U) / (du[:, :, None] * du[:, None, :]) / ANALYTIC_GATE
    ev = np.abs(g["V"] - blk.V) / (dv[:, :, None] * dv[:, None, :]) / ANALYTIC_GATE
    ew = np.abs(g["W"] - blk.W) / (du[P.cj][:, :, None] * dv[P.pi][:, None, :]) / ANALYTIC_GATE
    return {"U": float(eu.max()), "V": float(ev.max()), "W": float(ew.max())}


def fd_ratios(case):
    """cam_prep_kernel's perturbed rotations, the FD step rule and u_partial / u_final / v_kernel against the numpy forward
    differences, per entry over the propagated rounding bound of the differences (fd_block_bound)"""
    P, p, g = _case(*case, 0)
    A, B, eA, eB = rs.jacobian_fd(P, p, with_bound=True)
    blk = rs.normal_blocks(P, p, A, B, P.x - rs.evaluate(P, p))
    bU, bV, bW = fd_block_bound(P, A, B, eA, eB)
    return {key: float(np.max(np.abs(got - want) / np.maximum(bnd, 1e-300)))
            for key, got, want, bnd in (("U", g["U"], blk.U, bU), ("V", g["V"], blk.V, bV), ("W", g["W"], blk.W, bW))}


@pytest.mark.gpu
@pytest.mark.parametrize("case", BLOCK_CASES, ids=_ids)
def test_exported_S_equals_long_double_schur_of_exported_blocks(case):
    r = schur_ratios(case)
    assert max(r.values()) <= 1.0, (case, r)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BLOCK_CASES, ids=_ids)
def test_analytic_blocks_equal_exact_jacobian(case):
    """with rotation increments in both branches of (1 - cos)/theta^2, and camera and point constraints"""
    r = analytic_ratios(case)
    assert max(r.values()) <= 1.0, (case, r)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BLOCK_CASES, ids=_ids)
def test_fd_blocks_equal_numpy_forward_differences(case):
    r = fd_ratios(case)
    assert max(r.values()) <= 1.0, (case, r)


# ---- GPU: one LM iteration ---------------------------------------------------------------------------------------------
def _accepted(P, p, dp, mu, blk, p_eL2):
    pdp_eL2 = float(np.sum((P.x - rs.evaluate(P, p + dp)) ** 2)) + rs.penalty(P, p)
    eab = np.concatenate([blk.ea.reshape(-1), blk.eb.reshape(-1)])
    dL = float(np.sum(dp * (mu * dp + eab)))
    return dL > 0.0 and p_eL2 - pdp_eL2 > 0.0, pdp_eL2, dL


# relative gates of info[1] (error at p1), info[2] (|J^T e|_inf) and info[4] (mu_1 / maxdiag) in the analytic step test:
# info[1] and info[2] are sums over all observations of terms the two sides round differently (<= nvis u relative to the
# sum of |terms|, cancellation included); info[4] goes through dF / dL, a difference of two errors.
STEP_INFO_REL = (1e-9, 1e-9, 1e-6)


def analytic_step_ratios(name):
    """vinv_kernel, schur kernels with mu, the dense Cholesky, backsub_kernel and update_kernel: p1 of one accepted LM
    iteration in analytic mode against p0 + the restatement's damped step with the exact Jacobian.  Bound on the cameras:
    c u kappa(S + mu I) max|da| with c = (largest per-camera observation count + 100); on the points, that error
    propagated through V_i^-1 W_ij^T plus the same relative bound on db."""
    sc, kw = _step_problem(name)
    P = rs.problem(sc, **kw)
    p = P.p0
    rc, p1, info, _ = gpu_motstr(P, p, 1, 1)
    assert rc == 1 and int(info[7]) == 2 and int(info[9]) == 1, (name, rc, info)
    A, B = rs.jacobian_exact(P, p)
    e = P.x - rs.evaluate(P, p)
    return damped_step_ratios(P, p, p1, info, rs.normal_blocks(P, p, A, B, e), e, name)


def damped_step_ratios(P, p, p1, info, blk, e, name=""):
    """analytic_step_ratios' checks of p1 = the GPU's p after one accepted iteration from p, given the restatement's
    normal-equation blocks blk of the exact Jacobian and the residual e at p"""
    mu = 1e-3 * rs.max_diag(P, blk)
    S, E, Vinv = rs.schur(P, blk, mu)
    dp = rs.solve_reduced(P, blk, S, E, Vinv)
    p_eL2 = float(np.sum(e * e)) + rs.penalty(P, p)
    ok, pdp_eL2, dL = _accepted(P, p, dp, mu, blk, p_eL2)
    assert ok, name
    lam = np.linalg.eigvalsh(S)                       # S is SPD: cond_2(S) = lam_max / lam_min, without an SVD
    t = (np.bincount(P.cj).max() + 100) * u * (lam[-1] / lam[0])
    da, db = dp[:P.ncp], dp[P.ncp:].reshape(P.n, 3)
    gda, gdb = (p1 - p)[:P.ncp], (p1 - p)[P.ncp:].reshape(P.n, 3)
    sda = float(np.max(np.abs(da)))
    r = {"da": float(np.max(np.abs(gda - da)) / (t * sda + 2 * u * np.max(np.abs(p[:P.ncp]))))}
    Y = np.abs(blk.W @ Vinv[P.pi])                                       # |Y_ij| per observation
    G = np.zeros(P.n)
    np.add.at(G, P.pi, Y.sum(axis=(1, 2)))
    bnd = G[:, None] * t * sda + t * np.max(np.abs(db)) + 2 * u * np.abs(p[P.ncp:].reshape(P.n, 3))
    r["db"] = float(np.max(np.abs(gdb - db) / bnd))
    eab = np.concatenate([blk.ea.reshape(-1), blk.eb.reshape(-1)])
    tmp = 2.0 * (p_eL2 - pdp_eL2) / dL - 1.0
    mu1 = mu * max(1.0 - tmp ** 3, 0.3333333334)
    want = [pdp_eL2, float(np.max(np.abs(eab))), float(np.sum(dp * dp)), mu1 / rs.max_diag(P, blk)]
    tols = (STEP_INFO_REL[0], STEP_INFO_REL[1], 4 * t, STEP_INFO_REL[2])
    for q, w, tol in zip((1, 2, 3, 4), want, tols):
        r[f"info{q}"] = abs(info[q] - w) / (tol * abs(w))
    return r


def fd_step_ratios(name):
    """one accepted FD iteration against the unmodified reference run for exactly one iteration (REF_SBA_ITMAX = 1), over
    ten times the case's restatement-vs-reference spread (FD_SPREAD)"""
    from oracle import loader
    sc, kw = _step_problem(name)
    old = os.environ.get("REF_SBA_ITMAX")
    os.environ["REF_SBA_ITMAX"] = "1"
    try:
        ref = loader.run_sfm_ref(sc, **kw)
    finally:
        if old is None:
            del os.environ["REF_SBA_ITMAX"]
        else:
            os.environ["REF_SBA_ITMAX"] = old
    P = rs.problem(sc, **kw)
    rc, p1, info, _ = gpu_motstr(P, P.p0, 0, 1)
    assert rc == 1 and int(info[7]) == 2 and int(info[9]) == int(ref["info"][9]) == 1 and int(ref["info"][5]) == 1, (name, info)
    got = rs.unpack(P, p1)
    got["info"] = info
    return {"params": _step_spread(got, ref) / (10 * FD_SPREAD[name][0]), "info": _info_spread(got, ref) / (10 * FD_SPREAD[name][1])}


def mot_step_ratios(ef, ud, mcon):
    """mot_solve_kernel: one accepted motion-only iteration (analytic Jacobian) against (U_j + mu I) da_j = ea_j per camera
    with the exact Jacobian, camera constraints included; bound c u kappa(U_j + mu I) max|da_j| per camera, c as above"""
    sc = _complete_scene(1)
    cnp = 6 + ef + 2 * ud
    cons = constraints_for(sc, cnp, seed=9)
    cons.update(use_point_constraints=0, points_constraints=None, point_constraint_weight=0.0)
    P = rs.problem(sc, est_focal_length=ef, undistort=ud, ncons=mcon, **cons)
    a0 = P.p0[:P.ncp]
    rc, a1, info = gpu_mot(P, a0, 1, 1)
    assert rc == 1 and int(info[7]) == 2 and int(info[9]) == P.m - mcon, (rc, info)
    A, B = rs.jacobian_exact(P, P.p0)
    e = P.x - rs.evaluate(P, P.p0)
    blk = rs.normal_blocks(P, P.p0, A, B, e)
    mu = 1e-3 * float(np.max(np.diagonal(blk.U[mcon:], axis1=1, axis2=2)))
    da = rs.mot_step(P, blk, mu).reshape(P.m, cnp)
    got = (a1 - a0).reshape(P.m, cnp)
    assert np.array_equal(got[:mcon], np.zeros((mcon, cnp)))
    c = np.bincount(P.cj).max() + 100
    worst = 0.0
    for j in range(mcon, P.m):
        kap = np.linalg.cond(blk.U[j] + mu * np.eye(cnp))
        tol = c * u * kap * np.max(np.abs(da[j])) + 2 * u * np.max(np.abs(a0))
        worst = max(worst, float(np.max(np.abs(got[j] - da[j])) / tol))
    return {"da": worst}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STEP_CASES))
def test_one_analytic_iteration_equals_damped_step(name):
    r = analytic_step_ratios(name)
    assert max(r.values()) <= 1.0, (name, r)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STEP_CASES))
def test_one_fd_iteration_vs_reference(name):
    _ref_or_skip()
    r = fd_step_ratios(name)
    assert max(r.values()) <= 1.0, (name, r)


@pytest.mark.gpu
@pytest.mark.parametrize("ef,ud", MODES)
@pytest.mark.parametrize("mcon", [0, 2])
def test_one_motion_only_iteration_equals_per_camera_solve(ef, ud, mcon):
    r = mot_step_ratios(ef, ud, mcon)
    assert max(r.values()) <= 1.0, (ef, ud, mcon, r)
