"""numpy restatement of the reference's motion + structure BA, shared by the CPU and GPU tests.

The same restatement as oracle/ba_oracle.c (run_sfm, sfm.c:592-1003; sba_motstr_levmar_x, sba_levmar.c:457-2081; forward
differences, sba_levmar_wrap.c:163-259), in numpy, with the known_intrinsics branch of sfm_project_rd (sfm.c:339-357).
Dense Schur complement and LAPACK Cholesky (the reference's dpotrf); sums run in a different order than the reference's,
so results agree to rounding.  Motion + structure only (fix_points = 0), like ba_oracle.c.

The pieces of one LM iteration are separate functions, so that tests can compare one GPU kernel's output with its
restatement at a chosen point:
  - jacobian_fd: the reference's forward-difference Jacobian (its step rule), with a bound on its rounding error;
  - jacobian_exact: the exact Jacobian of the same projection, by complex-step differentiation;
  - normal_blocks: U / ea / V / eb / W with camera and point constraints and mcon fixed cameras;
  - schur: S = blockdiag(U + mu I) - W (V + mu I)^-1 W^T and E for a given mu;
  - solve_reduced / damped_step: one damped step dp;
  - port_run_sfm: the whole solve built on those."""
import types

import numpy as np

from bundler_sfm_b200 import bundle

F_SCALE, K_SCALE = 0.001, 5.0
U_ROUND = np.finfo(float).eps / 2


def rot_update_rows(R0, w):        # sfm.c:77-116 for every row of w (N x 3), R0 (N x 9); complex w for complex-step
    th = np.sqrt(w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1] + w[:, 2] * w[:, 2])
    out = R0.reshape(-1, 3, 3).astype(np.result_type(R0, w), copy=True)
    nz = th != 0.0
    if nz.any():
        n = w[nz] / th[nz, None]
        z = np.zeros(n.shape[0], n.dtype)
        nx = np.stack([z, -n[:, 2], n[:, 1], n[:, 2], z, -n[:, 0], -n[:, 1], n[:, 0], z], 1).reshape(-1, 3, 3)
        dR = np.eye(3)[None] + nx * np.sin(th[nz])[:, None, None] + (nx @ nx) * (1.0 - np.cos(th[nz]))[:, None, None]
        out[nz] = dR @ out[nz]
    return out.reshape(-1, 9)


def project_rows(a, b, R, f_fixed, kn, Kk, kk, est_focal, undistort, explicit_centers, f_scale=F_SCALE, k_scale=K_SCALE):
    """sfm_project_point3 for N observations: a (N x cnp), b (N x 3), R = rot_update(R_init, w) (N x 9).  The output has
    the inputs' dtype, so complex inputs give the complex-step derivative."""
    R = R.reshape(-1, 3, 3)
    if explicit_centers:
        bc = np.einsum("nij,nj->ni", R, b - a[:, 0:3])
    else:
        bc = np.einsum("nij,nj->ni", R, b) + a[:, 0:3]
    K0 = a[:, 6] / f_scale if est_focal else f_fixed
    p = np.empty((a.shape[0], 2), np.result_type(a, b, R))
    p[:, 0] = -bc[:, 0] * K0 / bc[:, 2]
    p[:, 1] = -bc[:, 1] * K0 / bc[:, 2]
    if kn.any():
        p[kn] = bundle.project_known(bc[kn], Kk[kn], kk[kn])
    if undistort:
        c = 7 if est_focal else 6
        k1, k2 = a[:, c] / k_scale, a[:, c + 1] / k_scale
        rsq = (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) / (K0 * K0)
        p *= (1.0 + k1 * rsq + k2 * rsq * rsq)[:, None]
    return p


def fd_step(v):                    # sba_levmar_wrap.c:207-212
    return np.maximum(np.abs(1e-4 * v), 1e-6)


def problem(scene, est_focal_length=1, undistort=1, explicit_camera_centers=1, ncons=0, use_constraints=0, constrained=None,
            constraints=None, weights=None, use_point_constraints=0, points_constraints=None, point_constraint_weight=0.0,
            known=None, K_known=None, k_known=None):
    """run_sfm's set-up (sfm.c:592-781): packing, constraint scaling, observation order -> namespace"""
    P = types.SimpleNamespace()
    P.vm = np.asarray(scene["vmask"]) != 0
    P.n, P.m = n, m = P.vm.shape
    P.est_focal, P.undistort, P.explicit_centers = est_focal_length, undistort, explicit_camera_centers
    P.cnp = cnp = 6 + (1 if est_focal_length else 0) + (2 if undistort else 0)
    P.ncp = m * cnp
    P.mcon = ncons
    P.pi, P.cj = np.nonzero(P.vm)                    # point-major, ascending camera (sba_levmar.c:652-663)
    P.nvis = len(P.pi)
    P.sel = P.cj >= P.mcon
    P.x = np.asarray(scene["projections"], float)
    P.R_init = np.asarray(scene["R"], float).reshape(m, 9)
    P.f_fixed = np.asarray(scene["f"], float)
    P.k_init = np.asarray(scene["k"], float)
    P.kn = np.zeros(m, bool) if known is None else np.asarray(known) != 0
    P.Kk = np.zeros((m, 9)) if K_known is None else np.asarray(K_known, float).reshape(m, 9)
    P.kk = np.zeros((m, 5)) if k_known is None else np.asarray(k_known, float).reshape(m, 5)
    a0 = np.zeros((m, cnp))                          # packing, sfm.c:652-703
    a0[:, 0:3] = scene["c"]
    if est_focal_length:
        a0[:, 6] = P.f_fixed * F_SCALE
    if undistort:
        c = 7 if est_focal_length else 6
        a0[:, c:c + 2] = P.k_init * K_SCALE
    P.p0 = np.concatenate([a0.reshape(-1), np.asarray(scene["pts"], float).reshape(-1)])
    P.nvars = P.p0.shape[0]
    P.use_constraints, P.use_point_constraints = use_constraints, use_point_constraints
    P.cc = np.zeros((m, cnp), bool); P.cv = np.zeros((m, cnp)); P.cw = np.zeros((m, cnp))
    if use_constraints:                              # sfm.c:721-754
        P.cc = np.asarray(constrained)[:, :cnp] != 0
        P.cv = np.asarray(constraints, float)[:, :cnp].copy(); P.cw = np.asarray(weights, float)[:, :cnp].copy()
        if est_focal_length:
            P.cv[:, 6] *= F_SCALE; P.cw[:, 6] *= 1.0 / (F_SCALE * F_SCALE)
        if undistort:
            c = 7 if est_focal_length else 6
            P.cv[:, c:c + 2] *= K_SCALE; P.cw[:, c:c + 2] *= 1.0 / (K_SCALE * K_SCALE)
    P.pc = np.zeros(n, bool); P.pv = np.zeros((n, 3))
    if use_point_constraints:                        # sfm.c:757-781
        P.pv = np.asarray(points_constraints, float)
        P.pc = ~np.all(P.pv == 0.0, axis=1)
    P.pw = point_constraint_weight
    return P


def penalty(P, pp):                                  # sba_levmar.c:808-842
    acc = 0.0
    if P.use_constraints:
        d = P.cv - pp[:P.ncp].reshape(P.m, P.cnp)
        acc += float(np.sum(np.where(P.cc, P.cw * d * d, 0.0)))
    if P.use_point_constraints:
        d = P.pv - pp[P.ncp:].reshape(P.n, 3)
        acc += float(np.sum(P.nvis * P.pw * d[P.pc] * d[P.pc]))
    return acc


def evaluate(P, pp, a=None, b=None, R=None):
    """predicted projections (nvis x 2) at pp; a / b / R override the per-observation camera, point and rotation rows"""
    A_ = pp[:P.ncp].reshape(P.m, P.cnp)[P.cj] if a is None else a
    B_ = pp[P.ncp:].reshape(P.n, 3)[P.pi] if b is None else b
    R_ = rot_update_rows(P.R_init[P.cj], A_[:, 3:6]) if R is None else R
    return project_rows(A_, B_, R_, P.f_fixed[P.cj], P.kn[P.cj], P.Kk[P.cj], P.kk[P.cj], P.est_focal, P.undistort,
                        P.explicit_centers)


def _obs_rows(P, p):
    a = p[:P.ncp].reshape(P.m, P.cnp)[P.cj]; b = p[P.ncp:].reshape(P.n, 3)[P.pi]
    return a, b, rot_update_rows(P.R_init[P.cj], a[:, 3:6])


def jacobian_fd(P, p, with_bound=False):
    """A (nvis x 2 x cnp), B (nvis x 2 x 3) by the reference's forward differences (sba_levmar_wrap.c:203-256).  With
    with_bound, also the per-entry rounding bound of a forward difference, u (|h(p + d)| + |h(p)| + 2 f) / d, without a
    constant: a projection is rounded relative to f |Pc| / |Pc_z| ~ f, not to |h|, which vanishes near the image centre."""
    a, b, R = _obs_rows(P, p)
    h0 = evaluate(P, p, a, b, R)
    f2 = 2.0 * (a[:, 6] / F_SCALE if P.est_focal else P.f_fixed[P.cj])[:, None]
    A = np.zeros((P.nvis, 2, P.cnp)); B = np.zeros((P.nvis, 2, 3))
    eA = np.zeros_like(A); eB = np.zeros_like(B)
    for jj in range(P.cnp):
        d = fd_step(a[:, jj]); a2 = a.copy(); a2[:, jj] = a[:, jj] + d
        R2 = rot_update_rows(P.R_init[P.cj], a2[:, 3:6]) if 3 <= jj <= 5 else R
        h1 = evaluate(P, p, a2, b, R2)
        A[:, :, jj] = (h1 - h0) * (1.0 / d)[:, None]
        eA[:, :, jj] = U_ROUND * (np.abs(h1) + np.abs(h0) + f2) / d[:, None]
    for jj in range(3):
        d = fd_step(b[:, jj]); b2 = b.copy(); b2[:, jj] = b[:, jj] + d
        h1 = evaluate(P, p, a, b2, R)
        B[:, :, jj] = (h1 - h0) * (1.0 / d)[:, None]
        eB[:, :, jj] = U_ROUND * (np.abs(h1) + np.abs(h0) + f2) / d[:, None]
    return (A, B, eA, eB) if with_bound else (A, B)


def jacobian_exact(P, p, h=1e-30):
    """the exact Jacobian of the same projection by complex-step differentiation: Im f(p + i h e_k) / h has no
    subtractive cancellation, so it is exact to rounding for any small h"""
    a, b, R = _obs_rows(P, p)
    A = np.zeros((P.nvis, 2, P.cnp)); B = np.zeros((P.nvis, 2, 3))
    for jj in range(P.cnp):
        a2 = a.astype(complex); a2[:, jj] += 1j * h
        R2 = rot_update_rows(P.R_init[P.cj], a2[:, 3:6]) if 3 <= jj <= 5 else R
        A[:, :, jj] = evaluate(P, p, a2, b, R2).imag / h
    for jj in range(3):
        b2 = b.astype(complex); b2[:, jj] += 1j * h
        B[:, :, jj] = evaluate(P, p, a, b2, R).imag / h
    return A, B


def normal_blocks(P, p, A, B, e):
    """U_j, ea_j (sba_levmar.c:932-964, camera constraints included, zero for j < mcon), V_i, eb_i (:987-1030, point
    constraints included) and W_ij = A_ij^T B_ij (zero for j < mcon, :1062-1065) -> namespace"""
    m, n, cnp, sel, pi, cj = P.m, P.n, P.cnp, P.sel, P.pi, P.cj
    U = np.zeros((m, cnp, cnp)); ea = np.zeros((m, cnp))
    np.add.at(U, cj[sel], np.einsum("oki,okj->oij", A[sel], A[sel]))
    np.add.at(ea, cj[sel], np.einsum("oki,ok->oi", A[sel], e[sel]))
    for j in range(P.mcon, m):                       # sba_levmar.c:952-963
        d = P.cv[j] - p[j * cnp:(j + 1) * cnp]
        U[j][np.diag_indices(cnp)] += np.where(P.cc[j], P.cw[j], 0.0)
        ea[j] += np.where(P.cc[j], P.cw[j] * d, 0.0)
    V = np.zeros((n, 3, 3)); eb = np.zeros((n, 3))
    np.add.at(V, pi, np.einsum("oki,okj->oij", B, B))
    np.add.at(eb, pi, np.einsum("oki,ok->oi", B, e))
    d = P.pv - p[P.ncp:].reshape(n, 3)
    V[P.pc] += (P.nvis * P.pw) * np.eye(3)[None]
    eb[P.pc] += P.nvis * P.pw * d[P.pc]
    W = np.einsum("oki,okj->oij", A, B)
    W[~sel] = 0.0
    return types.SimpleNamespace(U=U, ea=ea, V=V, eb=eb, W=W)


def max_diag(P, blk):                                # sba_levmar.c:1084-1116
    return max(np.finfo(float).tiny, float(np.max(np.diagonal(blk.U[P.mcon:], axis1=1, axis2=2), initial=0.0)),
               float(np.max(np.diagonal(blk.V, axis1=1, axis2=2))))


def schur(P, blk, mu):
    """S = blockdiag(U_j + mu I) - sum_i Y_ij W_ik^T over cameras >= mcon ((m - mcon) cnp square), E_j = ea_j - sum_i
    Y_ij eb_i, Y_ij = W_ij (V_i + mu I)^-1 (sba_levmar.c:1137-1338) -> (S, E, Vinv), or None when some V_i + mu I is
    singular (:1156-1161)"""
    m, n, cnp, mcon, sel, pi, cj = P.m, P.n, P.cnp, P.mcon, P.sel, P.pi, P.cj
    Vd = blk.V + mu * np.eye(3)[None]
    det = np.linalg.det(Vd)
    if not np.all(np.isfinite(det) & (det != 0.0)):
        return None
    Vinv = np.linalg.inv(Vd)
    Y = blk.W @ Vinv[pi]                              # Y_ij = W_ij V*_i^-1
    Sd = (m - mcon) * cnp
    S = np.zeros((m, cnp, m, cnp))
    for j in range(mcon, m):
        S[j, :, j, :] = blk.U[j] + mu * np.eye(cnp)
    E = blk.ea.copy()
    np.add.at(E, cj[sel], -np.einsum("oij,oj->oi", Y[sel], blk.eb[pi[sel]]))
    for i in range(n):                               # S_jk -= sum_i Y_ij W_ik^T
        os_ = np.nonzero((pi == i) & sel)[0]
        if len(os_):
            blkS = np.einsum("aik,bjk->aibj", Y[os_], blk.W[os_])
            S[np.ix_(cj[os_], range(cnp), cj[os_], range(cnp))] -= blkS
    return S[mcon:, :, mcon:, :].reshape(Sd, Sd), E[mcon:].reshape(-1), Vinv


def solve_reduced(P, blk, S, E, Vinv):
    """Cholesky solve of S da = E and the back substitution db_i = V*_i^-1 (eb_i - sum_j W_ij^T da_j) (:1340-1433)
    -> dp (nvars), or None when S is not positive definite"""
    try:
        L = np.linalg.cholesky(S)
        da = np.linalg.solve(L.T, np.linalg.solve(L, E))
    except np.linalg.LinAlgError:
        return None
    dp = np.zeros(P.nvars)
    dp[P.mcon * P.cnp:P.ncp] = da
    dacam = dp[:P.ncp].reshape(P.m, P.cnp)
    wt = np.zeros((P.n, 3))
    np.add.at(wt, P.pi[P.sel], np.einsum("oji,oj->oi", blk.W[P.sel], dacam[P.cj[P.sel]]))
    dp[P.ncp:] = np.einsum("nij,nj->ni", Vinv, blk.eb - wt).reshape(-1)
    return dp


def damped_step(P, blk, mu):
    """one damped step dp of the augmented normal equations, or None (singular V*_i or S not positive definite)"""
    sch = schur(P, blk, mu)
    return None if sch is None else solve_reduced(P, blk, *sch)


def mot_step(P, blk, mu):
    """motion-only step (sba_levmar.c:2487-2514): (U_j + mu I) da_j = ea_j per camera j >= mcon -> camera part of dp,
    or None when some U_j + mu I is not positive definite"""
    da = np.zeros((P.m, P.cnp))
    for j in range(P.mcon, P.m):
        try:
            L = np.linalg.cholesky(blk.U[j] + mu * np.eye(P.cnp))
        except np.linalg.LinAlgError:
            return None
        da[j] = np.linalg.solve(L.T, np.linalg.solve(L, blk.ea[j]))
    return da.reshape(-1)


def unpack(P, p):                                    # sfm.c:876-929
    a = p[:P.ncp].reshape(P.m, P.cnp)
    Rout = rot_update_rows(P.R_init, a[:, 3:6])
    f = a[:, 6] / F_SCALE if P.est_focal else P.f_fixed.copy()
    c = 7 if P.est_focal else 6
    k = a[:, c:c + 2] / K_SCALE if P.undistort else P.k_init.copy()
    return {"R": Rout, "c": a[:, 0:3].copy(), "f": f, "k": k, "pts": p[P.ncp:].reshape(P.n, 3).copy()}


def port_run_sfm(scene, eps2=1e-12, itmax=150, **kw):
    """run_sfm -> sba_motstr_levmar_x with forward differences; keywords as bundle.call_run_sfm.  Returns the unpacked
    solution with info[10], or None where the reference returns SBA_ERROR (almost singular normal equations)."""
    P = problem(scene, **kw)
    m, n, cnp, ncp, mcon = P.m, P.n, P.cnp, P.ncp, P.mcon
    p = P.p0.copy()
    opts = (1.0e-3, 1.0e-10, eps2, 1.0e-12, 0.0, 4.0e-2)           # sfm.c:705-714
    tau, eps1, eps2_, eps3_sq, eps4_sq, eps5 = abs(opts[0]), abs(opts[1]), abs(opts[2]), opts[3] ** 2, opts[4] ** 2, opts[5]
    eps2_sq = opts[2] * opts[2]
    e = P.x - evaluate(P, p)
    p_eL2 = float(np.sum(e * e)) + penalty(P, p)
    init_p_eL2 = p_eL2
    nfev, njev, nlss, stop, nu, mu, dp_L2, maxdiag, eab_inf = 1, 0, 0, 0, 2, 0.0, np.finfo(float).max, np.finfo(float).tiny, 0.0
    if not np.isfinite(p_eL2):
        stop = 7
    itno = 0
    while itno < itmax and not stop:
        A, B = jacobian_fd(P, p)
        njev += 1
        blk = normal_blocks(P, p, A, B, e)
        eab = np.concatenate([blk.ea.reshape(-1), blk.eb.reshape(-1)])
        eab_inf = float(np.max(np.abs(eab))); p_L2 = float(np.sum(p * p))
        maxdiag = max_diag(P, blk)
        if eab_inf <= eps1:
            dp_L2 = 0.0; stop = 1; break
        if itno == 0:
            mu = tau * maxdiag
        while True:                                  # damping loop, sba_levmar.c:1131-1597
            accepted = False
            sch = schur(P, blk, mu)
            if sch is None:
                pass                                 # singular V*_i: more damping (:1156-1161)
            else:
                nlss += 1
                dp = solve_reduced(P, blk, *sch)
                if dp is not None:
                    pdp = p + dp
                    dp_L2 = float(np.sum(dp * dp))
                    if dp_L2 <= eps2_sq * p_L2:
                        stop = 2; break
                    if dp_L2 >= (p_L2 + eps2_) / (1e-12 * 1e-12):
                        return None                  # almost singular: the reference returns SBA_ERROR
                    hx = P.x - evaluate(P, pdp); nfev += 1
                    pdp_eL2 = float(np.sum(hx * hx))
                    if not np.isfinite(pdp_eL2):
                        stop = 7; break
                    pdp_eL2 += penalty(P, p)         # constraint terms at the OLD p (:1487-1522)
                    dL = float(np.sum(dp * (mu * dp + eab)))
                    dF = p_eL2 - pdp_eL2
                    if dL > 0.0 and dF > 0.0:
                        tmp = 2.0 * dF / dL - 1.0
                        tmp = 1.0 - tmp * tmp * tmp
                        mu = mu * (tmp if tmp >= 0.3333333334 else 0.3333333334)
                        nu = 2
                        ef, hf = e.reshape(-1), hx.reshape(-1)
                        chk = ~((ef < eps5) & (hf < eps5))
                        with np.errstate(divide="ignore", invalid="ignore"):
                            pct = np.abs((ef[chk] - hf[chk]) / ef[chk])
                        max_pct = float(np.max(pct, initial=0.0))
                        if pdp_eL2 - 2.0 * np.sqrt(p_eL2 * pdp_eL2) < (eps4_sq - 1.0) * p_eL2:
                            stop = 4
                        if max_pct < eps5 and itno >= 4:
                            stop = 8; break
                        p, e, p_eL2 = pdp, hx, pdp_eL2
                        accepted = True
            if accepted:
                break
            mu *= nu                                 # :1584-1597 (int nu overflows after 2^30)
            if nu >= 1 << 30:
                stop = 6; break
            nu <<= 1
        if p_eL2 <= eps3_sq:
            stop = 5
        itno += 1
    if itno >= itmax:
        stop = 3
    info = np.array([init_p_eL2, p_eL2, eab_inf, dp_L2, mu / maxdiag, itno, stop, nfev, njev, nlss], float)
    out = unpack(P, p)
    out["info"] = info
    out["p"] = p
    return out
