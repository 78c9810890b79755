"""One LM step of reduced camera systems of more than 1536 unknowns, entry by entry, in the camera order the solver factors
in: the large Cholesky's panel path (apply_camera_order, the zero-block skip) and, above 4096 unknowns, the band path
(band_first_cols, chol_band_plan, chol_band_kernel, chol_backsolve_band_kernel), with schur_final_kernel writing S through
cam_block and backsub_kernel reading da back through it, mcon fixed cameras skipped.

The export pass writes S in the caller's order (ba_solver.cu: export_blocks sets cam_pos = nullptr), so S is never observed
in the order it is factored in.  And LM hides a wrong step: a block the envelope drops, or a permutation slip between
schur_final_kernel and backsub_kernel, still gives a step that goes downhill.  So every case checks the step itself:

- the camera-step residual S_mu da - E in long double, formed point by point from the GPU's own exported U, V and W
  without building S, over a bound made of the backward error of a Cholesky solve, the fp64 formation error of S and E, and
  the difference between the kernel's and the exact ea / eb.  It does not depend on the condition of S, so it holds at
  every size;
- the point-step residual W_i^T da + (V_i + mu I) db_i - eb_i of every point, and exact zeros for the fixed cameras;
- where cond(S) is affordable, the forward error of the step and info[1..4] (analytic_step_ratios of
  tests/test_ba_normal_equations.py); on one panel and one band case, the exported S against the long-double Schur
  complement of the exported blocks.

Each case first asserts the regime it is meant to test: on the CPU from the restatements (whether RCM is chosen, whether
the band plan fits), on the GPU also from the launch counts of bsfm_ba_chol_profile."""
import ctypes
import types

import numpy as np
import pytest
import scipy.sparse as sp

from bundler_sfm_b200 import bundle, synth
from tests import ba_restatement as rs
from tests import camera_order_restatement as R
from tests import chol_band_restatement as B
from tests.test_ba_camera_order import relabel_cameras
from tests.test_ba_normal_equations import (ANALYTIC_GATE, constraints_for, damped_step_ratios, gpu_motstr, graph_scene,
                                            schur_longdouble)

u = rs.U_ROUND
H100_WORKERS = {"H100 SXM": 131, "H100 PCIe": 113}      # SM count - 1: the band plan's worker CTAs
FORWARD_MAX_N = 4500        # cases up to this many unknowns also check the forward error (np.linalg.cond of the dense S)


def gamma(k):
    return k * u / (1.0 - k * u)


# ---- scenes ---------------------------------------------------------------------------------------------------------
def ring_graph(cams, reach=2, pair_pts=3, triple_pts=4):
    """graph_scene pairs / groups of a closed ring of cameras `cams`: each camera shares pair_pts two-view points with
    each of the next `reach` cameras, and triple_pts three-view points with the next two"""
    m = len(cams)
    pairs = [(cams[j], cams[(j + d) % m], pair_pts) for j in range(m) for d in range(1, reach + 1)]
    groups = [((cams[j], cams[(j + 1) % m], cams[(j + 2) % m]), triple_pts) for j in range(m)]
    return pairs, groups


def shuffled(m, seed):
    """cameras 0 .. m - 1 in a random order: a ring through them is far from banded in the natural order"""
    return [int(j) for j in np.random.default_rng(seed).permutation(m)]


def rcm_relabelled(scene):
    """the scene with its cameras numbered in RCM order: the solver then keeps the natural order"""
    m = len(scene["f"])
    pi, cj = np.nonzero(scene["vmask"])
    order = R.rcm(R.free_graph(R.scene_block_keys(pi, cj, m), m, 0))
    pos = np.empty(m, np.int64)
    pos[order] = np.arange(m)
    return relabel_cameras(scene, pos)


def _panel_ring250():        # the 250-camera strided ring of tests/test_ba_camera_order.py, cnp 9: 2250 unknowns
    sc = synth.ba_scene(250, 6000, 6, seed=250)
    sc["gt_pts"] = sc["pts"]
    return sc, {}


def _panel_natural():
    sc, kw = _panel_ring250()
    return rcm_relabelled(sc), kw


def _panel_mcon():           # 300 cameras, cnp 7, 3 fixed: 2079 unknowns
    pairs, groups = ring_graph(shuffled(300, seed=31))
    sc = graph_scene(300, pairs, groups, seed=31, explicit_centers=0)
    kw = dict(est_focal_length=1, undistort=0, explicit_camera_centers=0, ncons=3, **constraints_for(sc, 7, seed=3))
    return sc, kw


def _panel_wide():           # a random camera graph on a ring backbone, cnp 9: 4680 unknowns
    m = 520
    rng = np.random.default_rng(41)
    a, b = rng.integers(0, m, 700), rng.integers(0, m, 700)
    pairs = [(j, (j + 1) % m, 3) for j in range(m)] + [(int(x), int(y), 2) for x, y in zip(a, b) if x != y]
    groups = [((j, (j + 1) % m, (j + 2) % m), 3) for j in range(m)]
    return graph_scene(m, pairs, groups, seed=41), {}


def _band_ring():            # a closed ring of 500 cameras, cnp 9: 4500 unknowns
    pairs, groups = ring_graph(shuffled(500, seed=51))
    return graph_scene(500, pairs, groups, seed=51), {}


def _band_natural():
    sc, kw = _band_ring()
    return rcm_relabelled(sc), kw


def _band_mcon():            # 600 cameras, cnp 8, 5 fixed: 4760 unknowns
    pairs, groups = ring_graph(shuffled(600, seed=61))
    sc = graph_scene(600, pairs, groups, seed=61)
    kw = dict(est_focal_length=0, undistort=1, ncons=5, **constraints_for(sc, 8, seed=6))
    return sc, kw


COMPONENT_RING = 160         # 1440 rows at cnp 9: every component starts on a 32-row tile
LONE_CAMERAS = 4             # after the rings, sharing no point with any other camera


def _band_components():      # three disjoint rings of 160 cameras and four cameras alone, cnp 9: 4356 unknowns
    pairs, groups = [], []
    for r in range(3):
        p_, g_ = ring_graph([r * COMPONENT_RING + j for j in shuffled(COMPONENT_RING, seed=70 + r)])
        pairs += p_; groups += g_
    m = 3 * COMPONENT_RING + LONE_CAMERAS
    groups += [((j,), 6) for j in range(3 * COMPONENT_RING, m)]
    return graph_scene(m, pairs, groups, seed=71), {}


SINGLE_REACH = 3            # one point seen by cameras j and j + 3, for every other j: just past the ring's reach of 2


def _band_single_tuple():    # ring of 480 cameras, cnp 9: 4320 unknowns
    m = 480
    pairs, groups = ring_graph(list(range(m)))
    pairs += [(j, (j + SINGLE_REACH) % m, 1) for j in range(0, m, 2)]
    return graph_scene(m, pairs, groups, seed=81), {}


def _band_large():           # the config-3 camera graph (1000 cameras, strided ring) with 5000 points: 9000 unknowns
    sc = synth.ba_scene(1000, 5000, 6, seed=91)
    sc["gt_pts"] = sc["pts"]
    return sc, {}


# name: (scene maker, RCM chosen, band plan fits)
CASES = {
    "panel-rcm": (_panel_ring250, True, False),
    "panel-natural-kept": (_panel_natural, False, False),
    "panel-mcon-cons": (_panel_mcon, True, False),
    "panel-wide-above-4096": (_panel_wide, True, False),
    "band-rcm": (_band_ring, True, True),
    "band-natural": (_band_natural, False, True),
    "band-mcon-cons": (_band_mcon, True, True),
    "band-components": (_band_components, True, True),
    "band-single-tuple-reach": (_band_single_tuple, False, True),
    "band-large": (_band_large, True, True),
}

_SCENES = {}


def case_problem(name):
    """(scene, run_sfm keywords, restated problem) of a case, built once per session"""
    if name not in _SCENES:
        sc, kw = CASES[name][0]()
        _SCENES[name] = (sc, kw, rs.problem(sc, **kw))
    return _SCENES[name]


def regime(P, workers):
    """what the solver does with the problem P: (RCM chosen, cam_pos, band plan fits, first_col, block keys)"""
    keys = R.scene_block_keys(P.pi, P.cj, P.m, P.mcon)
    chosen, pos, _, _ = R.camera_order(keys, P.m, P.mcon, P.cnp)
    first = B.camera_first_cols(keys, P.m, P.mcon, P.cnp, pos)
    n = (P.m - P.mcon) * P.cnp
    fits = n > B.BAND_MIN_N and B.band_plan(first, n, workers)[0]
    return bool(chosen), pos, bool(fits), first, keys


def block_tuples(P):
    """tuples (shared points) of every camera pair j, k >= mcon, as a dense m x m count"""
    sel = P.sel
    vm = sp.csr_matrix((np.ones(int(sel.sum())), (P.pi[sel], P.cj[sel])), shape=(P.n, P.m))
    return (vm.T @ vm).toarray().astype(np.int64)


def one_tuple_first_rows(P, pos):
    """free cameras whose row's first column (lowest position among the camera and its neighbours) is set only by blocks
    of one tuple, in the order pos"""
    C = block_tuples(P)[P.mcon:, P.mcon:]
    pos = np.asarray(pos)
    out = []
    for v in range(C.shape[0]):
        nb = np.nonzero(C[v])[0]
        low = pos[nb].min()
        if low < pos[v]:
            setters = nb[pos[nb] == low]
            if np.all(C[v, setters] == 1):
                out.append(v)
    return out


# ---- the step residuals --------------------------------------------------------------------------------------------
def _inv3_longdouble(M):
    """inverse of every 3 x 3 block in long double (adjugate over determinant)"""
    r0, r1, r2 = M[:, 0, :], M[:, 1, :], M[:, 2, :]
    c0, c1, c2 = np.cross(r1, r2), np.cross(r2, r0), np.cross(r0, r1)
    det = np.einsum("na,na->n", r0, c0)
    return np.stack([c0, c1, c2], axis=2) / det[:, None, None]


def step_residuals(P, p, p1, g, blk, e):
    """The step p1 - p of one accepted LM iteration against the damped normal equations of the exported blocks g (U, V, W
    per observation; all cameras, as an mcon = 0 export gives them) and the exact ea / eb of blk, at the mu of the restated
    rule (1e-3 max diag of the GPU's U and V).  Camera rows: r = (U_j + mu I) da_j - ea_j - sum_i W_ij (V_i + mu I)^-1
    (sum_k W_ik^T da_k - eb_i), which is S_mu da - E, in long double without forming S.  Point rows: W_i^T da + (V_i + mu I)
    db_i - eb_i.  -> namespace: camera residuals (free cameras x cnp) and their bound, point residuals and their bound,
    the largest |da| of the fixed cameras."""
    ld = np.longdouble
    m, n, cnp, mcon = P.m, P.n, P.cnp, P.mcon
    sel = P.sel
    pi, cj = P.pi[sel], P.cj[sel]
    U, V, W = g["U"], g["V"], g["W"][sel]
    mu = 1e-3 * rs.max_diag(P, types.SimpleNamespace(U=U, V=V))
    dp = p1 - p
    da, db = dp[:P.ncp].reshape(m, cnp), dp[P.ncp:].reshape(n, 3)
    fixed = float(np.max(np.abs(da[:mcon]), initial=0.0))
    da = da.copy()
    da[:mcon] = 0.0
    I3, Ic = np.eye(3), np.eye(cnp)
    Vs = V + mu * I3
    X = _inv3_longdouble(V.astype(ld) + ld(mu) * I3)          # (V_i + mu I)^-1, long double
    Xa = np.abs(np.linalg.inv(Vs))
    kap = np.linalg.cond(Vs)
    Wa = np.abs(W)

    # residuals in long double
    Wl, dal = W.astype(ld), da.astype(ld)
    t = np.zeros((n, 3), ld)
    np.add.at(t, pi, np.einsum("oab,oa->ob", Wl, dal[cj]))    # sum_j W_ij^T da_j
    z = np.einsum("nab,nb->na", X, t - blk.eb.astype(ld))
    rc = np.einsum("jab,jb->ja", U.astype(ld) + ld(mu) * Ic, dal) - blk.ea.astype(ld)
    np.add.at(rc, cj, -np.einsum("oab,ob->oa", Wl, z[pi]))
    rc = rc[mcon:]
    rp = t + np.einsum("nab,nb->na", Vs.astype(ld), db.astype(ld)) - blk.eb.astype(ld)

    def abs_apply(x, wt):
        """(|U_j| + mu I) x_j + sum_i wt_i |W_ij| |(V_i + mu I)^-1| sum_k |W_ik|^T x_k, free camera rows"""
        y = np.zeros((n, 3))
        np.add.at(y, pi, np.einsum("oab,oa->ob", Wa, x[cj]))
        y = wt[:, None] * np.einsum("nab,nb->na", Xa, y)
        out = np.einsum("jab,jb->ja", np.abs(U) + mu * Ic, x)
        np.add.at(out, cj, np.einsum("oab,ob->oa", Wa, y[pi]))
        return out[mcon:]

    def through_points(y):
        """sum_i |W_ij| |(V_i + mu I)^-1| y_i, free camera rows"""
        out = np.zeros((m, cnp))
        np.add.at(out, cj, np.einsum("oab,ob->oa", Wa, np.einsum("nab,nb->na", Xa, y)[pi]))
        return out[mcon:]

    # diag(S_mu) for the Cholesky term: (|L| |L^T|)_ij <= sqrt(s_ii s_jj)
    Y = W @ np.linalg.inv(Vs)[pi]
    s = np.diagonal(U, axis1=1, axis2=2) + mu
    np.add.at(s, cj, -np.einsum("oab,oab->oa", Y, W))
    sq = np.sqrt(np.maximum(s[mcon:], 0.0))
    absda = np.abs(da)
    nsys = (m - mcon) * cnp
    b_chol = gamma(3 * nsys + 1) * sq * float(np.sum(sq * absda[mcon:]))
    # fp64 formation of S and E (schur_longdouble's summation bound, with the largest block's tuple count)
    nt = int(block_tuples(P).max())
    c = min(nt, 64) + (nt + 63) // 64 + 12
    b_form = c * u * (abs_apply(absda, kap) + np.abs(blk.ea[mcon:]) + through_points(kap[:, None] * np.abs(blk.eb)))
    # the kernel's ea / eb against the exact ones, at ANALYTIC_GATE of their Cauchy-Schwarz scale sqrt(U_aa) |e_j| (and the
    # constraint terms w d <= sqrt(U_aa) sqrt(w) |d|)
    e2 = (e * e).sum(1)
    ecam = np.sqrt(np.bincount(P.cj, weights=e2, minlength=m))
    ept = np.sqrt(np.bincount(P.pi, weights=e2, minlength=n))
    ccon = np.where(P.cc, np.sqrt(P.cw) * np.abs(P.cv - p[:P.ncp].reshape(m, cnp)), 0.0)
    pcon = np.where(P.pc[:, None], np.sqrt(P.nvis * P.pw) * np.abs(P.pv - p[P.ncp:].reshape(n, 3)), 0.0)
    dea = ANALYTIC_GATE * np.sqrt(np.diagonal(U, axis1=1, axis2=2)) * (ecam[:, None] + ccon)
    deb = ANALYTIC_GATE * np.sqrt(np.diagonal(V, axis1=1, axis2=2)) * (ept[:, None] + pcon)
    b_gate = dea[mcon:] + through_points(deb)
    # p1 - p is the step the GPU took to within u (|p1| + |step|)
    dl = u * (np.abs(p1[:P.ncp].reshape(m, cnp)) + absda)
    dl[:mcon] = 0.0
    dlp = u * (np.abs(p1[P.ncp:].reshape(n, 3)) + np.abs(db))
    b_round = abs_apply(dl, np.ones(n))
    bound_cam = b_chol + b_form + b_gate + b_round

    # points: db = fl(fl((V_i + mu I)^-1) fl(eb_i - sum_j W_ij^T da_j))
    WTda = np.zeros((n, 3))
    np.add.at(WTda, pi, np.einsum("oab,oa->ob", Wa, absda[cj]))
    nob = np.bincount(pi, minlength=n)
    err_g = gamma(cnp + nob + 1)[:, None] * (np.abs(blk.eb) + WTda)
    gabs = np.abs(blk.eb - t.astype(float)) + err_g
    VX = np.einsum("nab,nbc->nac", np.abs(Vs), Xa)
    b_pt = np.einsum("nab,nb->na", VX, ((12 * kap * u + gamma(3))[:, None] * gabs + err_g)) + deb
    WTdl = np.zeros((n, 3))
    np.add.at(WTdl, pi, np.einsum("oab,oa->ob", Wa, dl[cj]))
    b_pt += np.einsum("nab,nb->na", np.abs(Vs), dlp) + WTdl
    return types.SimpleNamespace(cam=rc, cam_bound=bound_cam, pt=rp, pt_bound=b_pt, fixed=fixed)


def step_residual_ratios(res):
    return {"camera": float(np.max(np.abs(res.cam).astype(float) / res.cam_bound)),
            "point": float(np.max(np.abs(res.pt).astype(float) / res.pt_bound))}


# ---- CPU: every case is in its regime ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_case_is_in_its_regime(name):
    """RCM chosen or not and the band plan fitting or not, as the case is meant to be, for the worker count of both H100
    models"""
    sc, kw, P = case_problem(name)
    want_rcm, want_band = CASES[name][1:]
    nsys = (P.m - P.mcon) * P.cnp
    assert nsys > R.LARGE_MIN
    assert (nsys > B.BAND_MIN_N) == (want_band or name == "panel-wide-above-4096")
    for model, workers in H100_WORKERS.items():
        chosen, pos, fits, first, keys = regime(P, workers)
        assert (chosen, fits) == (want_rcm, want_band), (model, chosen, fits)
    assert P.vm.sum(1).min() >= (1 if name == "band-components" else 2)
    if name == "band-components":      # the envelope restarts inside the system: row blocks that reach no earlier tile
        env = B.envelope(first, nsys)
        restarts = [rb for rb in range(1, len(env) - 1) if env[rb] == rb]
        assert restarts == [45, 90, 135], restarts      # the three components after the first; 135 is diagonal only
        assert env[136] == 135


def test_single_tuple_blocks_set_first_columns():
    """band-single-tuple-reach: in the order the solver factors in, many rows' first column is set only by blocks of one
    tuple (a camera pair sharing a single point), and without those blocks the envelope of the band plan would be
    narrower, so a band kernel that dropped them would lose a block of S"""
    sc, kw, P = case_problem("band-single-tuple-reach")
    chosen, pos, fits, first, keys = regime(P, H100_WORKERS["H100 SXM"])
    rows = one_tuple_first_rows(P, pos)
    assert len(rows) >= P.m // 4, len(rows)
    C = block_tuples(P)
    j, k = keys // P.m, keys % P.m
    thick = keys[(j == k) | (C[j, k] > 1)]
    nsys = P.m * P.cnp
    thin_first = B.camera_first_cols(thick, P.m, 0, P.cnp, pos)
    assert np.all(thin_first >= first) and np.any(B.envelope(thin_first, nsys) != B.envelope(first, nsys))


# ---- CPU: the sparse residual against a dense one -------------------------------------------------------------------
def _small_step(mcon):
    from tests.test_ba_normal_equations import _chunks_scene
    sc = _chunks_scene(1)
    P = rs.problem(sc, ncons=mcon, **constraints_for(sc, 9, seed=4))
    p = P.p0
    A, Bj = rs.jacobian_exact(P, p)
    e = P.x - rs.evaluate(P, p)
    blk = rs.normal_blocks(P, p, A, Bj, e)
    mu = 1e-3 * rs.max_diag(P, blk)
    S, E, Vinv = rs.schur(P, blk, mu)
    return P, p, e, blk, mu, S, E, Vinv


@pytest.mark.parametrize("mcon", [0, 2])
def test_sparse_residual_equals_dense_and_catches_a_dropped_block(mcon):
    """The point-by-point residual equals S_mu da - E of the dense long-double Schur complement, and LAPACK's step passes
    its gate.  The step of S with one off-diagonal block removed (the one-tuple block of cameras 0 and 1, or the 9-tuple
    block of cameras 2 and 4 when 0 and 1 are fixed) fails it by orders of magnitude."""
    P, p, e, blk, mu, S, E, Vinv = _small_step(mcon)
    g = dict(U=blk.U, V=blk.V, W=blk.W)
    p1 = p + rs.solve_reduced(P, blk, S, E, Vinv)
    res = step_residuals(P, p, p1, g, blk, e)
    r = step_residual_ratios(res)
    assert res.fixed == 0.0 and max(r.values()) <= 1.0, r
    # the dense residual in long double
    ld = np.longdouble
    I3, Ic = np.eye(3), np.eye(P.cnp)
    Sl, _ = schur_longdouble(P, blk.U + mu * Ic, blk.V + mu * I3, blk.W)
    X = _inv3_longdouble(blk.V.astype(ld) + ld(mu) * I3)
    El = blk.ea.astype(ld)
    np.add.at(El, P.cj, -np.einsum("oab,ob->oa", blk.W.astype(ld), np.einsum("nab,nb->na", X, blk.eb.astype(ld))[P.pi]))
    f = slice(mcon * P.cnp, P.ncp)
    dense = Sl[f, f] @ (p1 - p)[f].astype(ld) - El[mcon:].reshape(-1)
    assert np.max(np.abs(dense - res.cam.reshape(-1)).astype(float) / res.cam_bound.reshape(-1)) <= 1e-3
    # drop one block of S
    j, k = (0, 1) if mcon == 0 else (2, 4)
    assert block_tuples(P)[j, k] == (1 if mcon == 0 else 9)
    S2 = S.reshape(P.m - mcon, P.cnp, P.m - mcon, P.cnp).copy()
    S2[j - mcon, :, k - mcon, :] = 0.0
    S2[k - mcon, :, j - mcon, :] = 0.0
    p2 = p + rs.solve_reduced(P, blk, S2.reshape(S.shape), E, Vinv)
    bad = step_residual_ratios(step_residuals(P, p, p2, g, blk, e))
    assert bad["camera"] > 1e3, bad


# ---- GPU ------------------------------------------------------------------------------------------------------------
def device_workers():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count - 1


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _profiled_step(P, p):
    """one LM iteration (analytic Jacobian) with the large Cholesky's launch counts"""
    lib = bundle.load_library()
    lib.bsfm_ba_chol_profile.argtypes = [ctypes.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    lib.bsfm_ba_chol_profile(1)
    try:
        rc, p1, info, _ = gpu_motstr(P, p, 1, 1)
        ms, launches, fl = (ctypes.c_float * 4)(), (ctypes.c_int * 4)(), ctypes.c_double()
        lib.bsfm_ba_chol_profile_read(ms, launches, ctypes.byref(fl))
    finally:
        lib.bsfm_ba_chol_profile(0)
    return rc, p1, info, list(launches)


SCHUR_CASES = ("panel-rcm", "band-rcm")      # also: the exported S against the long-double Schur complement of the blocks


def large_step_ratios(name):
    """the regime of the case on this device, then the checks of one accepted LM iteration -> ratios (all <= 1 to pass)"""
    sc, kw, P = case_problem(name)
    want_rcm, want_band = CASES[name][1:]
    workers = device_workers()
    chosen, pos, fits, first, keys = regime(P, workers)
    assert (chosen, fits) == (want_rcm, want_band), (name, chosen, fits)
    p = P.p0
    P0 = types.SimpleNamespace(**vars(P))         # U, V, W export (mcon = 0: the export covers every camera)
    P0.mcon, P0.sel = 0, np.ones_like(P.sel)
    rc0, _, _, g = gpu_motstr(P0, p, 1, 0, export=True)
    assert rc0 == 0, (name, rc0, bundle.load_library().bsfm_last_error())
    rc, p1, info, launches = _profiled_step(P, p)
    assert rc == 1 and int(info[7]) == 2 and int(info[9]) == 1, (name, rc, info)
    if want_band:
        assert launches[0] == 1 and launches[1] == 0 and launches[2] == 0, (name, launches)
    else:
        assert launches[1] > 0 and launches[2] > 0, (name, launches)
    A, Bj = rs.jacobian_exact(P, p)
    e = P.x - rs.evaluate(P, p)
    blk = rs.normal_blocks(P, p, A, Bj, e)
    res = step_residuals(P, p, p1, g, blk, e)
    assert res.fixed == 0.0, (name, res.fixed)
    r = step_residual_ratios(res)
    nsys = (P.m - P.mcon) * P.cnp
    if nsys <= FORWARD_MAX_N:
        r.update(damped_step_ratios(P, p, p1, info, blk, e, name))
    if name in SCHUR_CASES:
        S, bound = schur_longdouble(P0, g["U"], g["V"], g["W"])
        r["S"] = float(np.max(np.abs(g["S"].astype(np.longdouble) - S).astype(float) / np.maximum(bound, 1e-300)))
    print(f"\n{name}: {nsys} unknowns, {workers} workers, RCM {'chosen' if chosen else 'not chosen'}, band plan "
          f"{'fits' if fits else 'does not fit'}, launches {launches} ({'band' if want_band else 'panel'} path); "
          + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    return r


@pytest.mark.gpu
@pytest.mark.skipif(not _has_gpu(), reason="needs a CUDA device")
@pytest.mark.parametrize("name", list(CASES))
def test_large_step_solves_the_damped_normal_equations(name):
    r = large_step_ratios(name)
    assert max(r.values()) <= 1.0, (name, r)
