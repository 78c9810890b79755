// ba_kernels.cu -- sm_90a kernels of the BA hot path (fp64).  Compiled with -fmad=false so the
// projection keeps the reference's un-fused operation order (gcc x86-64 does not contract).
//
// Reference loops restated as kernels (file:line under /root/reference):
//   K1 residual      sba_motstr_Qs          lib/sba-1.5/sba_levmar_wrap.c:73-104
//                    sfm_project_point3     lib/sfm-driver/sfm.c:503-552
//                    sfm_project_rd         lib/sfm-driver/sfm.c:302-380
//                    rot_update             lib/sfm-driver/sfm.c:77-116
//                    sfm_project_point2_fisheye  lib/sfm-driver/sfm.c:448-492 (FE kernels; sfm_project2 :243-299,
//                                           sfm_fisheye_distort :426-446)
//   K2 Jacobian      sba_motstr_Qs_fdjac    lib/sba-1.5/sba_levmar_wrap.c:163-259  (FD mode)
//                    snavely_reprojection_error.h:58-92 / SURVEY.md A.4            (analytic mode)
//   K3 U,ea / V,eb / W                      lib/sba-1.5/sba_levmar.c:919-964 / 987-1030 / 1053-1082
//   K4 (V+mu I)^-1                          lib/sba-1.5/sba_levmar.c:1137-1162
//   K5 Schur S, E                           lib/sba-1.5/sba_levmar.c:1170-1339
//   K7 back-substitution                    lib/sba-1.5/sba_levmar.c:1393-1433
//   K8 norms / gain / stop-8                lib/sba-1.5/sba_levmar.c:1084-1128, 1443-1561
#include "ba_kernels.cuh"
#include <cfloat>

namespace bsfm {
namespace ba {

// ------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}

// Deterministic grid reduction: every block writes its partial, the last block to finish (ticket)
// combines the partials in block order.  `op` 0 = sum, 1 = max.  Returns true in thread 0 of the
// last block with the final value in `out`.
template <int OP>
__device__ bool grid_reduce(double v, double *partial, unsigned int *ticket, double &out)
{
    __shared__ double sm[32];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();   // protects sm[] / is_last when a kernel calls grid_reduce more than once
    v = OP == 0 ? warp_sum(v) : warp_max(v);
    if (lane == 0) sm[wid] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double acc = sm[0];
        for (int w = 1; w < nw; w++) acc = OP == 0 ? acc + sm[w] : fmax(acc, sm[w]);
        partial[blockIdx.x] = acc;
        __threadfence();
        unsigned int t = atomicAdd(ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return false;
    __threadfence();
    // last block: fixed-order combine (thread-strided then tree inside the block; deterministic)
    double acc = OP == 0 ? 0.0 : -DBL_MAX;
    for (int b = threadIdx.x; b < (int) gridDim.x; b += blockDim.x) {
        double pv = ((volatile double *) partial)[b];
        acc = OP == 0 ? acc + pv : fmax(acc, pv);
    }
    acc = OP == 0 ? warp_sum(acc) : warp_max(acc);
    __syncthreads();
    if (lane == 0) sm[wid] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = sm[0];
        for (int w = 1; w < nw; w++) r = OP == 0 ? r + sm[w] : fmax(r, sm[w]);
        out = r;
        *ticket = 0;
        return true;
    }
    return false;
}

// rot_update, lib/sfm-driver/sfm.c:77-116 (Rodrigues about the initial rotation)
__device__ void rot_update_dev(const double *R, double w0, double w1, double w2, double *Rn)
{
    const double theta = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
    if (theta == 0.0) {
#pragma unroll
        for (int q = 0; q < 9; q++) Rn[q] = R[q];
        return;
    }
    const double n0 = w0 / theta, n1 = w1 / theta, n2 = w2 / theta;
    double nx[9] = {0.0, -n2, n1, n2, 0.0, -n0, -n1, n0, 0.0};
    double nxsq[9];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) nxsq[3 * r + c] = nx[3 * r] * nx[c] + nx[3 * r + 1] * nx[3 + c] + nx[3 * r + 2] * nx[6 + c];
    const double sinth = sin(theta), costh = cos(theta);
    const double omc = 1.0 - costh;
    double dR[9];
#pragma unroll
    for (int q = 0; q < 9; q++) {
        const double ident = (q == 0 || q == 4 || q == 8) ? 1.0 : 0.0;
        const double term2 = nx[q] * sinth;
        const double term3 = nxsq[q] * omc;
        dR[q] = (ident + term2) + term3;
    }
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) Rn[3 * r + c] = dR[3 * r] * R[c] + dR[3 * r + 1] * R[3 + c] + dR[3 * r + 2] * R[6 + c];
}

// finite-difference step, lib/sba-1.5/sba_levmar_wrap.c:207-212 (SBA_DELTA_SCALE, SBA_MIN_DELTA)
__device__ __forceinline__ double fd_step(double v)
{
    double d = 1E-04 * v;
    d = fabs(d);
    if (d < 1E-06) d = 1E-06;
    return d;
}

// sfm_project_point3 + sfm_project_rd (lib/sfm-driver/sfm.c:503-552, 302-380).  KI = false: every camera takes the
// known_intrinsics = 0 branch and `ci` is not read.  KI = true: calibrated cameras (ci->known) take the other branch;
// the radial step after it is the same for both and still uses the focal parameter K0.
// FE = true: sfm_project_point2_fisheye (sfm.c:448-492) instead: the same pinhole (sfm_project2, :243-299) without the
// radial step, then the fisheye mapping for cameras with cf->fisheye (sfm_fisheye_distort, :426-446).  FE = false never
// reads `cf`.
template <bool KI, bool FE>
__device__ __forceinline__ void project_dev(const Model &M, const CamIntrinsics *ci, const CamFisheye *cf, const double (&a)[MAX_CNP],
                                            const double *R, double f_fixed, double b0, double b1, double b2, double &px, double &py)
{
    double bc0, bc1, bc2;
    if (M.explicit_centers) {
        const double d0 = b0 - a[0], d1 = b1 - a[1], d2 = b2 - a[2];
        bc0 = R[0] * d0 + R[1] * d1 + R[2] * d2;
        bc1 = R[3] * d0 + R[4] * d1 + R[5] * d2;
        bc2 = R[6] * d0 + R[7] * d1 + R[8] * d2;
    } else {
        bc0 = R[0] * b0 + R[1] * b1 + R[2] * b2;
        bc1 = R[3] * b0 + R[4] * b1 + R[5] * b2;
        bc2 = R[6] * b0 + R[7] * b1 + R[8] * b2;
        bc0 += a[0]; bc1 += a[1]; bc2 += a[2];
    }
    const double K0 = M.est_focal ? a[6] / M.f_scale : f_fixed;
    double p0, p1;
    if (KI && ci->known) {
        project_known_dev(*ci, bc0, bc1, bc2, p0, p1);
    } else {
        p0 = -bc0 * K0 / bc2;
        p1 = -bc1 * K0 / bc2;
    }
    if (FE) {
        if (cf->fisheye) fisheye_distort_dev(*cf, p0, p1, p0, p1);
    } else if (M.undistort) {
        const double k1 = (M.est_focal ? a[7] : a[6]) / M.k_scale;
        const double k2 = (M.est_focal ? a[8] : a[7]) / M.k_scale;
        const double rsq = (p0 * p0 + p1 * p1) / (K0 * K0);
        const double factor = 1.0 + k1 * rsq + k2 * rsq * rsq;
        p0 *= factor;
        p1 *= factor;
    }
    px = p0; py = p1;
}

__device__ __forceinline__ void load_cam(const Problem &P, const double *p, int j, double (&a)[MAX_CNP])
{
#pragma unroll
    for (int q = 0; q < MAX_CNP; q++) a[q] = (q < P.M.cnp) ? p[(size_t) j * P.M.cnp + q] : 0.0;
}

// ------------------------------------------------------------------------------------------------
// camera prep: R(w) and, for the FD Jacobian, R(w + d e_k) k=0..2 (sfm.c:539-547 recomputes the
// cached rotation whenever w changes, i.e. for each perturbed w component)
// ------------------------------------------------------------------------------------------------
__global__ void cam_prep_kernel(Problem P, const double *p, int with_pert)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P.m) return;
    const double *a = p + (size_t) j * P.M.cnp;
    const double *R0 = P.R_init + (size_t) j * 9;
    double Rn[9];
    rot_update_dev(R0, a[3], a[4], a[5], Rn);
#pragma unroll
    for (int q = 0; q < 9; q++) P.camR[(size_t) j * 36 + q] = Rn[q];
    if (with_pert) {
        for (int k = 0; k < 3; k++) {
            double w[3] = {a[3], a[4], a[5]};
            w[k] = w[k] + fd_step(w[k]);
            rot_update_dev(R0, w[0], w[1], w[2], Rn);
#pragma unroll
            for (int q = 0; q < 9; q++) P.camR[(size_t) j * 36 + 9 * (k + 1) + q] = Rn[q];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K1: e = x - f(p), sum e^2 (sba_levmar.c:802-806, nrmL2xmy :159-207)
// also: stop-8 statistic against a previous residual vector when e_prev != nullptr (:1552-1561)
// ------------------------------------------------------------------------------------------------
template <bool KI, bool FE>
__global__ void residual_kernel(Problem P, const double *p, double *e_out, const double *e_prev, double eps5)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    double s = 0.0, pct = 0.0;
    if (o < P.nvis) {
        const int j = P.obs_cam[o], i = P.obs_pt[o];
        double a[MAX_CNP];
        load_cam(P, p, j, a);
        const double *b = p + (size_t) P.m * P.M.cnp + (size_t) i * 3;
        double hx, hy;
        project_dev<KI, FE>(P.M, KI ? P.intr + j : nullptr, FE ? P.fe + j : nullptr, a, P.camR + (size_t) j * 36, P.f_fixed[j],
                            b[0], b[1], b[2], hx, hy);
        const double e0 = P.x[2 * (size_t) o] - hx, e1 = P.x[2 * (size_t) o + 1] - hy;
        e_out[2 * (size_t) o] = e0;
        e_out[2 * (size_t) o + 1] = e1;
        s = e0 * e0 + e1 * e1;
        if (e_prev) {
            const double q0 = e_prev[2 * (size_t) o], q1 = e_prev[2 * (size_t) o + 1];
            if (!(q0 < eps5 && e0 < eps5)) pct = fabs((q0 - e0) / q0);
            if (!(q1 < eps5 && e1 < eps5)) { const double c = fabs((q1 - e1) / q1); if (c > pct) pct = c; }
        }
    }
    double out;
    if (grid_reduce<0>(s, P.partial, P.ticket, out)) {
        P.sc->e_L2 = out;
        P.sc->nonfinite = isfinite(out) ? 0 : 1;
    }
    if (e_prev) {
        // NaN pct (0/0 cannot occur: both < eps5 is skipped) ; inf stays inf
        if (grid_reduce<1>(pct, P.partial + gridDim.x, P.ticket + 1, out)) P.sc->max_pct = out;
    }
}
template __global__ void residual_kernel<false, false>(Problem, const double *, double *, const double *, double);
template __global__ void residual_kernel<true, false>(Problem, const double *, double *, const double *, double);
template __global__ void residual_kernel<false, true>(Problem, const double *, double *, const double *, double);
template __global__ void residual_kernel<true, true>(Problem, const double *, double *, const double *, double);

// ------------------------------------------------------------------------------------------------
// K2 + W of K3: per observation A_ij (2 x cnp), B_ij (2 x 3), W_ij = A^T B (cnp x 3)
// ------------------------------------------------------------------------------------------------
template <bool KI, bool FE>
__device__ __forceinline__ void analytic_jac(const Problem &P, const CamIntrinsics *ci, const CamFisheye *cf, const double (&a)[MAX_CNP],
                                             const double *R0, double f_fixed, double b0, double b1, double b2, double (&A)[2][MAX_CNP],
                                             double (&B)[2][3])
{
    // SURVEY.md A.4.  v = R_init (X - c) [or R_init X], Pc = exp([w]x) v (+ t), q = -Pc.xy / Pc.z
    const Model &M = P.M;
    const double w0 = a[3], w1 = a[4], w2 = a[5];
    double R[9];
    rot_update_dev(R0, w0, w1, w2, R);
    double X0 = b0, X1 = b1, X2 = b2;
    if (M.explicit_centers) { X0 -= a[0]; X1 -= a[1]; X2 -= a[2]; }
    double Pc0 = R[0] * X0 + R[1] * X1 + R[2] * X2;
    double Pc1 = R[3] * X0 + R[4] * X1 + R[5] * X2;
    double Pc2 = R[6] * X0 + R[7] * X1 + R[8] * X2;
    // rotated part (without translation) is what d/dw acts on
    const double Pr0 = Pc0, Pr1 = Pc1, Pr2 = Pc2;
    if (!M.explicit_centers) { Pc0 += a[0]; Pc1 += a[1]; Pc2 += a[2]; }
    // the fisheye projection has no radial step: its k columns are zero
    const bool radial = M.undistort && !FE;
    const double f = M.est_focal ? a[6] / M.f_scale : f_fixed;
    const double k1 = radial ? (M.est_focal ? a[7] : a[6]) / M.k_scale : 0.0;
    const double k2 = radial ? (M.est_focal ? a[8] : a[7]) / M.k_scale : 0.0;
    const double iz = 1.0 / Pc2;
    const double q0 = -Pc0 * iz, q1 = -Pc1 * iz;
    double G[2][3];
    double Ai[2][3];   // calibrated camera: columns of f*f_scale, k1*k_scale, k2*k_scale (sfm.c:673-681)
    double rho, r;
    double ph0, ph1;   // the pinhole projection, what the fisheye mapping acts on
    if (KI && ci->known) {
        // calibrated camera: u = Kc d(q) (Brown-Conrady d, Kc = [[K0, K1], [0, K4]]), then the radial step
        // xhat = u (1 + k1 s + k2 s^2), s = |u|^2 / f^2.  dxhat/dq = (fac I + h u u^T) Kc Jd, h = 2 (k1 + 2 k2 s) / f^2
        const double *kd = ci->k, *Kc = ci->K;
        const double rsq = q0 * q0 + q1 * q1;
        const double F = 1.0 + kd[0] * rsq + kd[1] * rsq * rsq + kd[4] * rsq * rsq * rsq;
        const double dF = kd[0] + 2.0 * kd[1] * rsq + 3.0 * kd[4] * rsq * rsq;
        const double xd = q0 * F + 2.0 * kd[2] * q0 * q1 + kd[3] * (rsq + 2.0 * q0 * q0);
        const double yd = q1 * F + kd[2] * (rsq + 2.0 * q1 * q1) + 2.0 * kd[3] * q0 * q1;
        // Jd = d(xd, yd)/d(q0, q1) (symmetric)
        const double J00 = F + 2.0 * q0 * q0 * dF + 2.0 * kd[2] * q1 + 6.0 * kd[3] * q0;
        const double J01 = 2.0 * q0 * q1 * dF + 2.0 * kd[2] * q0 + 2.0 * kd[3] * q1;
        const double J11 = F + 2.0 * q1 * q1 * dF + 6.0 * kd[2] * q1 + 2.0 * kd[3] * q0;
        const double M00 = Kc[0] * J00 + Kc[1] * J01, M01 = Kc[0] * J01 + Kc[1] * J11;
        const double M10 = Kc[3] * J01, M11 = Kc[3] * J11;
        const double u0 = Kc[0] * xd + Kc[1] * yd + Kc[2], u1 = Kc[3] * yd + Kc[4];
        ph0 = u0; ph1 = u1;
        // without the radial step f is not read at all (it may be unset when it is not estimated either)
        const double s = radial ? (u0 * u0 + u1 * u1) / (f * f) : 0.0;
        const double fac = 1.0 + k1 * s + k2 * s * s;
        const double h = radial ? 2.0 * (k1 + 2.0 * k2 * s) / (f * f) : 0.0;
        const double P00 = fac + h * u0 * u0, P01 = h * u0 * u1, P11 = fac + h * u1 * u1;
        const double D00 = P00 * M00 + P01 * M10, D01 = P00 * M01 + P01 * M11;
        const double D10 = P01 * M00 + P11 * M10, D11 = P01 * M01 + P11 * M11;
        G[0][0] = -iz * D00; G[0][1] = -iz * D01; G[0][2] = -iz * (D00 * q0 + D01 * q1);
        G[1][0] = -iz * D10; G[1][1] = -iz * D11; G[1][2] = -iz * (D10 * q0 + D11 * q1);
        // the focal length enters only through s (zero column without the radial step)
        const double dsf = radial ? -2.0 * s / f * (k1 + 2.0 * k2 * s) : 0.0;
        const double uu[2] = {u0, u1};
#pragma unroll
        for (int k = 0; k < 2; k++) {
            Ai[k][0] = uu[k] * dsf / M.f_scale;
            Ai[k][1] = uu[k] * s / M.k_scale;
            Ai[k][2] = uu[k] * s * s / M.k_scale;
        }
    } else {
        rho = q0 * q0 + q1 * q1;
        r = 1.0 + k1 * rho + k2 * rho * rho;
        const double g = 2.0 * (k1 + 2.0 * k2 * rho);
        // dxhat/dq (2x2) = f ( r I + g q q^T )
        const double D00 = f * (r + g * q0 * q0), D01 = f * g * q0 * q1, D11 = f * (r + g * q1 * q1);
        // dq/dPc (2x3) = -(1/z) [ I | q ]
        // G = dxhat/dPc (2x3)
        G[0][0] = -iz * D00; G[0][1] = -iz * D01; G[0][2] = -iz * (D00 * q0 + D01 * q1);
        G[1][0] = -iz * D01; G[1][1] = -iz * D11; G[1][2] = -iz * (D01 * q0 + D11 * q1);
        ph0 = f * q0; ph1 = f * q1;
    }
    // fisheye mapping x_d = g(|u|) u + c of the pinhole output u, g(r) = s atan(r / F) / r, s = (180 / pi) f_rad / (f_angle / 2):
    // dx_d/du = g I + (g'(r) / r) u u^T, g'(r) / r = (s / (F (1 + (r / F)^2)) - g) / r^2
    double Jf00 = 1.0, Jf01 = 0.0, Jf11 = 1.0;
    const bool fish = FE && cf->fisheye;
    if (fish) {
        const double rr = ph0 * ph0 + ph1 * ph1, rf = sqrt(rr);
        const double sc = (180.0 / BSFM_M_PI) * cf->rad / (0.5 * cf->angle);
        const double x = rf / cf->focal;
        const double g = sc * atan(x) / rf;
        const double gp = (sc / (cf->focal * (1.0 + x * x)) - g) / rr;
        Jf00 = g + gp * ph0 * ph0; Jf01 = gp * ph0 * ph1; Jf11 = g + gp * ph1 * ph1;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const double g0 = G[0][c], g1 = G[1][c];
            G[0][c] = Jf00 * g0 + Jf01 * g1;
            G[1][c] = Jf01 * g0 + Jf11 * g1;
        }
    }
    // B = G R ; dPc/dc = -R (explicit centres) or dPc/dt = I
#pragma unroll
    for (int k = 0; k < 2; k++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
            B[k][c] = G[k][0] * R[c] + G[k][1] * R[3 + c] + G[k][2] * R[6 + c];
            A[k][c] = M.explicit_centers ? -B[k][c] : G[k][c];
        }
    // dPr/dw = -[Pr]x J_l(w)
    const double th2 = w0 * w0 + w1 * w1 + w2 * w2;
    double ca, cb;   // (1-cos)/th^2, (th - sin)/th^3
    if (th2 < 1e-8) { ca = 0.5 - th2 / 24.0; cb = 1.0 / 6.0 - th2 / 120.0; }
    else { const double th = sqrt(th2); ca = (1.0 - cos(th)) / th2; cb = (th - sin(th)) / (th2 * th); }
    const double wx[9] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0};
    double Jl[9];
#pragma unroll
    for (int rr = 0; rr < 3; rr++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const double wx2 = wx[3 * rr] * wx[c] + wx[3 * rr + 1] * wx[3 + c] + wx[3 * rr + 2] * wx[6 + c];
            Jl[3 * rr + c] = ((rr == c) ? 1.0 : 0.0) + ca * wx[3 * rr + c] + cb * wx2;
        }
    // M3 = -[Pr]x = [[0, Pr2, -Pr1], [-Pr2, 0, Pr0], [Pr1, -Pr0, 0]]
    const double M3[9] = {0.0, Pr2, -Pr1, -Pr2, 0.0, Pr0, Pr1, -Pr0, 0.0};
    double dPdw[9];
#pragma unroll
    for (int rr = 0; rr < 3; rr++)
#pragma unroll
        for (int c = 0; c < 3; c++) dPdw[3 * rr + c] = M3[3 * rr] * Jl[c] + M3[3 * rr + 1] * Jl[3 + c] + M3[3 * rr + 2] * Jl[6 + c];
#pragma unroll
    for (int k = 0; k < 2; k++)
#pragma unroll
        for (int c = 0; c < 3; c++) A[k][3 + c] = G[k][0] * dPdw[c] + G[k][1] * dPdw[3 + c] + G[k][2] * dPdw[6 + c];
    // intrinsics
    const double qq[2] = {q0, q1};
    double dfs_v[2];
#pragma unroll
    for (int k = 0; k < 2; k++) dfs_v[k] = (KI && ci->known) ? Ai[k][0] : r * qq[k] / M.f_scale;
    if (fish) {
        const double d0 = dfs_v[0], d1 = dfs_v[1];
        dfs_v[0] = Jf00 * d0 + Jf01 * d1;
        dfs_v[1] = Jf01 * d0 + Jf11 * d1;
    }
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const bool kn = KI && ci->known;
        const double dfs = dfs_v[k];
        const double dk1 = FE ? 0.0 : (kn ? Ai[k][1] : f * rho * qq[k] / M.k_scale);
        const double dk2 = FE ? 0.0 : (kn ? Ai[k][2] : f * rho * rho * qq[k] / M.k_scale);
        A[k][6] = M.est_focal ? dfs : (M.undistort ? dk1 : 0.0);
        A[k][7] = M.est_focal ? (M.undistort ? dk1 : 0.0) : (M.undistort ? dk2 : 0.0);
        A[k][8] = (M.est_focal && M.undistort) ? dk2 : 0.0;
    }
}

template <bool KI, bool FE>
__global__ void __launch_bounds__(128) jacobian_kernel(Problem P, const double *p, int jac_mode)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= P.nvis) return;
    const Model &M = P.M;
    const int cnp = M.cnp;
    const int j = P.obs_cam[o], i = P.obs_pt[o];
    double a[MAX_CNP];
    load_cam(P, p, j, a);
    const double *bp = p + (size_t) P.m * cnp + (size_t) i * 3;
    double b[3] = {bp[0], bp[1], bp[2]};
    const double ff = P.f_fixed[j];
    const CamIntrinsics *ci = KI ? P.intr + j : nullptr;
    const CamFisheye *cf = FE ? P.fe + j : nullptr;
    double A[2][MAX_CNP], B[2][3];

    if (jac_mode == 1) {
        analytic_jac<KI, FE>(P, ci, cf, a, P.R_init + (size_t) j * 9, ff, b[0], b[1], b[2], A, B);
    } else {
        const double *Rb = P.camR + (size_t) j * 36;
        double h0, h1;
        project_dev<KI, FE>(M, ci, cf, a, Rb, ff, b[0], b[1], b[2], h0, h1);
#pragma unroll
        for (int jj = 0; jj < MAX_CNP; jj++) {
            A[0][jj] = 0.0; A[1][jj] = 0.0;
            if (jj < cnp) {
                const double d = fd_step(a[jj]);
                const double d1 = 1.0 / d;
                const double tmp = a[jj];
                a[jj] = tmp + d;
                const double *R = (jj >= 3 && jj <= 5) ? (Rb + 9 * (jj - 2)) : Rb;
                double g0, g1;
                project_dev<KI, FE>(M, ci, cf, a, R, ff, b[0], b[1], b[2], g0, g1);
                a[jj] = tmp;
                A[0][jj] = (g0 - h0) * d1;
                A[1][jj] = (g1 - h1) * d1;
            }
        }
#pragma unroll
        for (int jj = 0; jj < 3; jj++) {
            const double d = fd_step(b[jj]);
            const double d1 = 1.0 / d;
            const double tmp = b[jj];
            b[jj] = tmp + d;
            double g0, g1;
            project_dev<KI, FE>(M, ci, cf, a, Rb, ff, b[0], b[1], b[2], g0, g1);
            b[jj] = tmp;
            B[0][jj] = (g0 - h0) * d1;
            B[1][jj] = (g1 - h1) * d1;
        }
    }
    double *jA = P.jacA + (size_t) o * 2 * cnp;
    double *jB = P.jacB + (size_t) o * 6;
    double *Wo = P.W + (size_t) o * cnp * 3;
    const bool fixed_cam = j < P.mcon;   // A_ij assumed zero (sba_levmar.c:1062-1065)
#pragma unroll
    for (int ii = 0; ii < MAX_CNP; ii++) {
        if (ii < cnp) {
            jA[ii] = A[0][ii];
            jA[cnp + ii] = A[1][ii];
#pragma unroll
            for (int jj = 0; jj < 3; jj++) {
                double sum = 0.0;
                sum += A[0][ii] * B[0][jj];
                sum += A[1][ii] * B[1][jj];
                Wo[ii * 3 + jj] = fixed_cam ? 0.0 : sum;
            }
        }
    }
#pragma unroll
    for (int jj = 0; jj < 3; jj++) { jB[jj] = B[0][jj]; jB[3 + jj] = B[1][jj]; }
}
template __global__ void jacobian_kernel<false, false>(Problem, const double *, int);
template __global__ void jacobian_kernel<true, false>(Problem, const double *, int);
template __global__ void jacobian_kernel<false, true>(Problem, const double *, int);
template __global__ void jacobian_kernel<true, true>(Problem, const double *, int);

// ------------------------------------------------------------------------------------------------
// K3: V_i, eb_i -- one thread per point, observations in ascending camera order (same summation
// order as sba_levmar.c:987-1030)
// ------------------------------------------------------------------------------------------------
__global__ void v_kernel(Problem P, const double *p, const double *e)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    double V[6] = {0, 0, 0, 0, 0, 0};   // 00 01 02 11 12 22
    double eb[3] = {0, 0, 0};
    for (int o = P.rowptr[i]; o < P.rowptr[i + 1]; o++) {
        const double *B = P.jacB + (size_t) o * 6;
        const double b00 = B[0], b01 = B[1], b02 = B[2], b10 = B[3], b11 = B[4], b12 = B[5];
        const double e0 = e[2 * (size_t) o], e1 = e[2 * (size_t) o + 1];
        double s;
        s = 0.0; s += b00 * b00; s += b10 * b10; V[0] += s;
        s = 0.0; s += b00 * b01; s += b10 * b11; V[1] += s;
        s = 0.0; s += b00 * b02; s += b10 * b12; V[2] += s;
        s = 0.0; s += b01 * b01; s += b11 * b11; V[3] += s;
        s = 0.0; s += b01 * b02; s += b11 * b12; V[4] += s;
        s = 0.0; s += b02 * b02; s += b12 * b12; V[5] += s;
        s = 0.0; s += b00 * e0; s += b10 * e1; eb[0] += s;
        s = 0.0; s += b01 * e0; s += b11 * e1; eb[1] += s;
        s = 0.0; s += b02 * e0; s += b12 * e1; eb[2] += s;
    }
    if (P.pt_constrained && P.pt_constrained[i]) {   // sba_levmar.c:1017-1029
        const double w = (double) P.nvis * P.pt_weights[i];
        const double *b = p + (size_t) P.m * P.M.cnp + (size_t) i * 3;
        const double d0 = P.pt_constraints[3 * (size_t) i] - b[0];
        const double d1 = P.pt_constraints[3 * (size_t) i + 1] - b[1];
        const double d2 = P.pt_constraints[3 * (size_t) i + 2] - b[2];
        V[0] += w; V[3] += w; V[5] += w;
        eb[0] += w * d0; eb[1] += w * d1; eb[2] += w * d2;
    }
    double *Vo = P.V + (size_t) i * 9;
    Vo[0] = V[0]; Vo[1] = V[1]; Vo[2] = V[2];
    Vo[3] = V[1]; Vo[4] = V[3]; Vo[5] = V[4];
    Vo[6] = V[2]; Vo[7] = V[4]; Vo[8] = V[5];
    double *ebo = P.eab + (size_t) P.m * P.M.cnp + (size_t) i * 3;
    ebo[0] = eb[0]; ebo[1] = eb[1]; ebo[2] = eb[2];
}

// ------------------------------------------------------------------------------------------------
// K3: U_j, ea_j -- one CTA per camera; threads stride over the camera's observations, then a
// fixed-shape tree (warp shuffles + shared memory) combines them: deterministic.
// ------------------------------------------------------------------------------------------------
constexpr int U_THREADS = 128;
// pass 1: CTA (j, seg) accumulates the seg-th slice of camera j's observations -> Upart[j][seg][54]
__global__ void __launch_bounds__(U_THREADS) u_partial_kernel(Problem P, const double *e, int nseg)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int j = blockIdx.x / nseg, seg = blockIdx.x % nseg;
    const int cnp = P.M.cnp;
    double acc[54];   // 45 upper-triangular U entries (row-major) + 9 ea
#pragma unroll
    for (int q = 0; q < 54; q++) acc[q] = 0.0;
    if (j >= P.mcon) {
        const int c0 = P.cam_ptr[j], c1 = P.cam_ptr[j + 1];
        const int len = (c1 - c0 + nseg - 1) / nseg;
        const int s0 = c0 + seg * len, s1 = min(c1, s0 + len);
        for (int t = s0 + threadIdx.x; t < s1; t += U_THREADS) {
            const int o = P.cam_obs[t];
            const double *jA = P.jacA + (size_t) o * 2 * cnp;
            double A0[MAX_CNP], A1[MAX_CNP];
#pragma unroll
            for (int q = 0; q < MAX_CNP; q++) { A0[q] = (q < cnp) ? jA[q] : 0.0; A1[q] = (q < cnp) ? jA[cnp + q] : 0.0; }
            const double e0 = e[2 * (size_t) o], e1 = e[2 * (size_t) o + 1];
            int q = 0;
#pragma unroll
            for (int ii = 0; ii < MAX_CNP; ii++)
#pragma unroll
                for (int jj = ii; jj < MAX_CNP; jj++) { double sv = 0.0; sv += A0[ii] * A0[jj]; sv += A1[ii] * A1[jj]; acc[q++] += sv; }
#pragma unroll
            for (int ii = 0; ii < MAX_CNP; ii++) { double sv = 0.0; sv += A0[ii] * e0; sv += A1[ii] * e1; acc[45 + ii] += sv; }
        }
    }
    __shared__ double sm[U_THREADS / 32][54];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < 54; q++) {
        double v = warp_sum(acc[q]);
        if (lane == 0) sm[wid][q] = v;
    }
    __syncthreads();
    if (threadIdx.x < 54) {
        double v = sm[0][threadIdx.x];
        for (int w = 1; w < U_THREADS / 32; w++) v += sm[w][threadIdx.x];
        P.u_part[((size_t) j * nseg + seg) * 54 + threadIdx.x] = v;
    }
}

// pass 2: combine the segments in order, scatter to U_j (full symmetric) and ea_j, add constraints
__global__ void __launch_bounds__(96) u_final_kernel(Problem P, const double *p, int nseg)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    __shared__ double sm[54];
    const int j = blockIdx.x;
    const int cnp = P.M.cnp;
    if (threadIdx.x < 54) {
        double v = 0.0;
        for (int sgm = 0; sgm < nseg; sgm++) v += P.u_part[((size_t) j * nseg + sgm) * 54 + threadIdx.x];
        sm[threadIdx.x] = v;
    }
    __syncthreads();
    if (threadIdx.x < 81) {
        const int ii = threadIdx.x / 9, jj = threadIdx.x % 9;
        if (ii < cnp && jj < cnp) {
            const int r = ii < jj ? ii : jj, c = ii < jj ? jj : ii;
            const int q = r * 9 - r * (r - 1) / 2 + (c - r);
            double v = sm[q];
            if (ii == jj && P.cam_constrained && j >= P.mcon && P.cam_constrained[(size_t) j * cnp + ii])
                v += P.cam_weights[(size_t) j * cnp + ii];     // sba_levmar.c:952-963
            P.U[(size_t) j * cnp * cnp + ii * cnp + jj] = v;
        }
    } else if (threadIdx.x < 90) {
        const int ii = threadIdx.x - 81;
        if (ii < cnp) {
            double v = sm[45 + ii];
            if (P.cam_constrained && j >= P.mcon && P.cam_constrained[(size_t) j * cnp + ii]) {
                const double diff = P.cam_constraints[(size_t) j * cnp + ii] - p[(size_t) j * cnp + ii];
                v += P.cam_weights[(size_t) j * cnp + ii] * diff;
            }
            P.eab[(size_t) j * cnp + ii] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K8a: ||J^T e||_inf, ||p||^2, max diagonal (sba_levmar.c:1084-1128) and constraint penalty
// (:808-842).  Single CTA, fixed order.
// ------------------------------------------------------------------------------------------------
__global__ void grad_stats_kernel(Problem P, const double *p)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int cnp = P.M.cnp;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    double inf = 0.0, pl2 = 0.0, md = DBL_MIN;
    if (q < P.nlm) {
        inf = fabs(P.eab[q]);
        pl2 = p[q] * p[q];
        if (q < P.m * cnp) {
            const int j = q / cnp, ii = q % cnp;
            if (j >= P.mcon) md = P.U[(size_t) j * cnp * cnp + ii * cnp + ii];
        } else {
            const int r = q - P.m * cnp;
            md = P.V[(size_t) (r / 3) * 9 + (r % 3) * 4];
        }
    }
    double out;
    if (grid_reduce<1>(inf, P.partial, P.ticket, out)) P.sc->eab_inf = out;
    if (grid_reduce<0>(pl2, P.partial + gridDim.x, P.ticket + 1, out)) P.sc->p_L2 = out;
    if (grid_reduce<1>(md, P.partial + 2 * gridDim.x, P.ticket + 2, out)) P.sc->max_diag = fmax(out, DBL_MIN);
}

__global__ void penalty_kernel(Problem P, const double *p)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    // evaluated by one thread in the reference's order (small: m*cnp + constrained points)
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int cnp = P.M.cnp;
    double pen = 0.0;
    if (P.cam_constrained) {
        for (int j = 0; j < P.m; j++)
            for (int jj = 0; jj < cnp; jj++)
                if (P.cam_constrained[(size_t) j * cnp + jj]) {
                    const double diff = P.cam_constraints[(size_t) j * cnp + jj] - p[(size_t) j * cnp + jj];
                    pen += P.cam_weights[(size_t) j * cnp + jj] * diff * diff;
                }
    }
    if (P.pt_constrained) {
        for (int i = 0; i < P.n; i++)
            if (P.pt_constrained[i])
                for (int ii = 0; ii < 3; ii++) {
                    const double diff = P.pt_constraints[3 * (size_t) i + ii] - p[(size_t) P.m * cnp + (size_t) i * 3 + ii];
                    pen += P.nvis * P.pt_weights[i] * diff * diff;
                }
    }
    P.sc->penalty = pen;
}

// ------------------------------------------------------------------------------------------------
// K4: (V_i + mu I)^-1, 3x3 SPD via Cholesky (reference: LAPACK dsytrf/dsytri, sba_lapack.c:1053-1140)
// ------------------------------------------------------------------------------------------------
__global__ void vinv_kernel(Problem P)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const double mu = *P.mu;
    const double *V = P.V + (size_t) i * 9;
    const double a00 = V[0] + mu, a01 = V[1], a02 = V[2], a11 = V[4] + mu, a12 = V[5], a22 = V[8] + mu;
    // cofactor inverse of a symmetric 3x3 (exact formula; the matrix is SPD for mu > 0)
    const double c00 = a11 * a22 - a12 * a12;
    const double c01 = a02 * a12 - a01 * a22;
    const double c02 = a01 * a12 - a02 * a11;
    const double det = a00 * c00 + a01 * c01 + a02 * c02;
    if (!(det != 0.0) || !isfinite(det)) { P.sc->singular_v = 1; return; }
    const double id = 1.0 / det;
    const double c11 = a00 * a22 - a02 * a02;
    const double c12 = a01 * a02 - a00 * a12;
    const double c22 = a00 * a11 - a01 * a01;
    double *O = P.Vinv + (size_t) i * 9;
    O[0] = c00 * id; O[1] = c01 * id; O[2] = c02 * id;
    O[3] = c01 * id; O[4] = c11 * id; O[5] = c12 * id;
    O[6] = c02 * id; O[7] = c12 * id; O[8] = c22 * id;
}

// ------------------------------------------------------------------------------------------------
// K5: S_jk = delta_jk (U_j + mu I) - sum_i Y_ij W_ik^T,  E_j = ea_j - sum_i Y_ij eb_i,
// Y_ij = W_ij (V_i + mu I)^-1   (sba_levmar.c:1195-1338).
// Upper blocks (j <= k) only; every block's tuple list (ascending point = the reference's summation
// order) is cut into chunks of SCHUR_CHUNK tuples.  Pass A: one warp per chunk accumulates a partial
// 9x9 (+ 9 for E on diagonal blocks).  Pass B: one warp per block adds its chunks in order and writes
// S (both triangles) and E.  Fixed shapes and orders => bitwise reproducible.
// ------------------------------------------------------------------------------------------------
// The 9x3 . 3x9 products run on the fp64 tensor cores: Y_ij (rows padded to 16, K padded to 4) is the A
// operand of mma.sync.m8n8k4.f64, W_ik^T the B operand; column 9 of the second n-tile carries eb_i, so the
// E_j partial sum comes out of the same instruction.  Every lane forms its own fragment elements straight
// from global memory (the 27-double blocks are L1-resident), so there are no shuffles.
__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// Operand staging of schur_partial_kernel.  With the operands of ONE tuple in flight per warp (a register double buffer) the kernel
// is bound by bytes in flight, not by HBM, so in-flight data lives in shared memory: every warp keeps SCHUR_DEPTH tuples' operand blocks
// (W_ij 27 + W_ik 27 + Vinv_i 9 + eb_i 3 doubles) on their way with cp.async (8-byte granules: the 216-byte W blocks are only
// 8-byte aligned), and forms its MMA fragments from shared memory.  Same arithmetic, same order: bitwise the same partial sums.
constexpr int SCHUR_DEPTH = 8;
constexpr int SCHUR_STAGE = 68;          // doubles per staged tuple (66 used)
__device__ __forceinline__ void cp_async8(double *smem_dst, const double *gsrc)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t) __cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(128) schur_partial_kernel(Problem P)
{
    __shared__ double stage_all[4][SCHUR_DEPTH][SCHUR_STAGE];
    __shared__ int4 rec_all[4][SCHUR_CHUNK];
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (c >= P.nchunks) return;
    double (*stage)[SCHUR_STAGE] = stage_all[threadIdx.x >> 5];
    const int cnp = P.M.cnp, m = P.m;
    // block of this chunk: last b with chunk_off[b] <= c
    int lo = 0, hi = P.nblocks - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (P.chunk_off[mid] <= c) lo = mid; else hi = mid - 1; }
    const int b = lo;
    const uint32_t key = P.blk_key[b];
    const bool diag = (key / (uint32_t) m) == (key % (uint32_t) m);
    const int t0 = P.blk_start[b] + (c - P.chunk_off[b]) * SCHUR_CHUNK;
    const int t1 = min(t0 + SCHUR_CHUNK, P.blk_start[b + 1]);
    const int nY = cnp * 3;
    const int g = lane >> 2, tg = lane & 3;
    const bool kv = tg < 3;                       // K = 3 padded to 4
    const bool r0v = kv && g < cnp;               // A rows 0..7
    const bool r1v = kv && 8 + g < cnp;           // A rows 8..15 (only row 8 exists for cnp = 9)
    const bool c0v = kv && g < cnp;               // B cols 0..7
    const bool c1v = kv && 8 + g < cnp;           // B cols 8..15
    const bool ev = kv && diag && g == 1;         // B col 9 <- eb_i
    const double *eb = P.eab + (size_t) m * cnp;
    double a00[2] = {0, 0}, a01[2] = {0, 0}, a10[2] = {0, 0}, a11[2] = {0, 0};

    // the chunk's tuple records (<= 64) go to shared memory once; every lane then knows, for each of its (at most three) 8-byte
    // slots of a tuple's operand block, WHICH record component indexes it, the array it comes from and the stride -- all fixed
    // for the whole chunk, so issuing a tuple is one shared-memory load, one multiply-add and one cp.async per slot instead of a
    // selection among four pointers per element (the kernel is bound by instruction issue)
    static_assert(SCHUR_CHUNK <= 64, "64 tuple records per warp");
    int4 *recs = rec_all[threadIdx.x >> 5];
    for (int q = lane; q < t1 - t0; q += 32) recs[q] = P.tuples[t0 + q];
    // operand block layout: [0, nY) W_ij, [nY, 2 nY) W_ik, [2 nY, 2 nY + 9) Vinv_i, then eb_i (3)
    const int oW2 = nY, oV = 2 * nY, oE = 2 * nY + 9, nElem = 2 * nY + 12;
    const double *sbase[3];
    int sstride[3], scomp[3];
    bool sval[3];
#pragma unroll
    for (int q = 0; q < 3; q++) {
        const int e = lane + 32 * q;
        sval[q] = e < nElem;
        if (e < oW2)      { sbase[q] = P.W + e;             sstride[q] = nY; scomp[q] = 0; }
        else if (e < oV)  { sbase[q] = P.W + (e - oW2);     sstride[q] = nY; scomp[q] = 1; }
        else if (e < oE)  { sbase[q] = P.Vinv + (e - oV);   sstride[q] = 9;  scomp[q] = 2; }
        else              { sbase[q] = eb + (e - oE);       sstride[q] = 3;  scomp[q] = 2; }
    }
    __syncwarp();
    const int *reci = reinterpret_cast<const int *>(recs);
    auto issue = [&](int i /* tuple index inside the chunk */) {
        double *dst = stage[i % SCHUR_DEPTH] + lane;
#pragma unroll
        for (int q = 0; q < 3; q++)
            if (sval[q]) cp_async8(dst + 32 * q, sbase[q] + (size_t) reci[4 * i + scomp[q]] * sstride[q]);
    };
    const int nt = t1 - t0;
    for (int d = 0; d < SCHUR_DEPTH; d++) {
        if (d < nt) issue(d);
        cp_async_commit();
    }
    for (int i = 0; i < nt; i++) {
        cp_async_wait<SCHUR_DEPTH - 1>();            // this lane's part of tuple i has landed ...
        __syncwarp();                               // ... and everybody else's
        const double *S = stage[i % SCHUR_DEPTH];
        double wa0[3] = {0, 0, 0}, wa1[3] = {0, 0, 0}, vi[3] = {0, 0, 0};
        if (kv) { vi[0] = S[oV + tg]; vi[1] = S[oV + 3 + tg]; vi[2] = S[oV + 6 + tg]; }
        if (r0v) { wa0[0] = S[g * 3]; wa0[1] = S[g * 3 + 1]; wa0[2] = S[g * 3 + 2]; }
        if (r1v) { wa1[0] = S[(8 + g) * 3]; wa1[1] = S[(8 + g) * 3 + 1]; wa1[2] = S[(8 + g) * 3 + 2]; }
        const double bb0 = c0v ? S[oW2 + g * 3 + tg] : 0.0;
        const double bb1 = c1v ? S[oW2 + (8 + g) * 3 + tg] : (ev ? S[oE + tg] : 0.0);
        // Y[row][tg] = sum_c Wa[row][c] * Vinv[c][tg]   (sba_levmar.c:1206-1214)
        double y0 = 0.0, y1 = 0.0;
        y0 += wa0[0] * vi[0]; y0 += wa0[1] * vi[1]; y0 += wa0[2] * vi[2];
        y1 += wa1[0] * vi[0]; y1 += wa1[1] * vi[1]; y1 += wa1[2] * vi[2];
        if (!r0v) y0 = 0.0;
        if (!r1v) y1 = 0.0;
        // YWt += Y W_ik^T  (sba_levmar.c:1262-1275), E partial in column 9 (:1318-1333)
        dmma884(a00[0], a00[1], y0, bb0);
        dmma884(a01[0], a01[1], y0, bb1);
        dmma884(a10[0], a10[1], y1, bb0);
        dmma884(a11[0], a11[1], y1, bb1);
        __syncwarp();                               // the stage is free again
        if (i + SCHUR_DEPTH < nt) issue(i + SCHUR_DEPTH);
        cp_async_commit();
    }
    // accumulator element (row = g, col = 2 tg + e) of tile (mt, nt) -> entry (mt*8 + g, nt*8 + 2 tg + e)
    double *out = P.schur_part + (size_t) c * SCHUR_PART_STRIDE;
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int col0 = 2 * tg + e, col1 = 8 + 2 * tg + e;
        if (g < cnp) {
            if (col0 < cnp) out[g * cnp + col0] = a00[e];
            if (col1 < cnp) out[g * cnp + col1] = a01[e];
            else if (diag && col1 == 9) out[81 + g] = a01[e];
        }
        if (8 + g < cnp) {
            if (col0 < cnp) out[(8 + g) * cnp + col0] = a10[e];
            if (col1 < cnp) out[(8 + g) * cnp + col1] = a11[e];
            else if (diag && col1 == 9) out[81 + 8 + g] = a11[e];
        }
    }
}

__global__ void __launch_bounds__(128) schur_final_kernel(Problem P)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= P.nblocks) return;
    const int cnp = P.M.cnp, m = P.m, nn = cnp * cnp;
    const double mu = *P.mu;
    const uint32_t key = P.blk_key[b];
    const int j = (int) (key / (uint32_t) m), k = (int) (key % (uint32_t) m);
    const int c0 = P.chunk_off[b], c1 = P.chunk_off[b + 1];
    double acc[3] = {0.0, 0.0, 0.0}, accE = 0.0;
    for (int c = c0; c < c1; c += 4) {
        // four chunks' partials are fetched together, then added in chunk order (deterministic)
        double v[4][4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const bool ok = c + u < c1;
            const double *part = P.schur_part + (size_t) (ok ? c + u : c) * SCHUR_PART_STRIDE;
#pragma unroll
            for (int rep = 0; rep < 3; rep++) { const int q = lane + 32 * rep; v[u][rep] = (ok && q < nn) ? part[q] : 0.0; }
            v[u][3] = (ok && j == k && lane < cnp) ? part[81 + lane] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) { acc[0] += v[u][0]; acc[1] += v[u][1]; acc[2] += v[u][2]; accE += v[u][3]; }
    }
    const int Sdim = P.Sdim;
    const int jr = cam_block(P, j) * cnp, kr = cam_block(P, k) * cnp;      // S is symmetric: both triangles are written
#pragma unroll
    for (int rep = 0; rep < 3; rep++) {
        const int q = lane + 32 * rep;
        if (q < nn) {
            const int ii = q / cnp, jj = q % cnp;
            double v;
            if (j == k) {
                double u = P.U[(size_t) j * nn + ii * cnp + jj];
                if (ii == jj) u += mu;
                v = u - acc[rep];
            } else {
                v = -acc[rep];
            }
            P.S[(size_t) (jr + ii) * Sdim + (kr + jj)] = v;
            if (j != k) P.S[(size_t) (kr + jj) * Sdim + (jr + ii)] = v;
        }
    }
    if (j == k && lane < cnp) P.E[jr + lane] = P.eab[(size_t) j * cnp + lane] - accE;
}

// zero the dense S (blocks of camera pairs with no common point stay zero)
__global__ void zero_kernel(double *ptr, size_t count)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    size_t q = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t) gridDim.x * blockDim.x;
    for (; q < count; q += stride) ptr[q] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// K7: db_i = (V_i+mu I)^-1 (eb_i - sum_j W_ij^T da_j)   (sba_levmar.c:1393-1433); also fills dp for
// the camera part from the dense solution `da` (zero for j < mcon, :1378)
// ------------------------------------------------------------------------------------------------
__global__ void backsub_kernel(Problem P, const double *da)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int cnp = P.M.cnp;
    if (i < P.m * cnp) {
        const int j = i / cnp;
        P.dp[i] = (j < P.mcon) ? 0.0 : da[cam_block(P, j) * cnp + (i - j * cnp)];
    }
    if (i >= P.n) return;
    double w0 = 0.0, w1 = 0.0, w2 = 0.0;
    for (int o = P.rowptr[i]; o < P.rowptr[i + 1]; o++) {
        const int j = P.obs_cam[o];
        if (j < P.mcon) continue;
        const double *Wo = P.W + (size_t) o * cnp * 3;
        const double *d = da + (size_t) cam_block(P, j) * cnp;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int jj = 0; jj < cnp; jj++) {
            const double dv = d[jj];
            s0 += Wo[jj * 3 + 0] * dv; s1 += Wo[jj * 3 + 1] * dv; s2 += Wo[jj * 3 + 2] * dv;
        }
        w0 += s0; w1 += s1; w2 += s2;
    }
    const double *eb = P.eab + (size_t) P.m * cnp + (size_t) i * 3;
    w0 = eb[0] - w0; w1 = eb[1] - w1; w2 = eb[2] - w2;
    const double *Vi = P.Vinv + (size_t) i * 9;
    double *db = P.dp + (size_t) P.m * cnp + (size_t) i * 3;
#pragma unroll
    for (int ii = 0; ii < 3; ii++) {
        double s = 0.0;
        s += Vi[ii * 3 + 0] * w0; s += Vi[ii * 3 + 1] * w1; s += Vi[ii * 3 + 2] * w2;
        db[ii] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// motion-only BA (sba_mot_levmar_x, sba_levmar.c:2495-2514): the augmented normal equations are block diagonal,
// (U_j + mu I) da_j = ea_j per camera, solved like sba_Axb_Chol (Cholesky, failure on a non-positive pivot).
// One thread per camera (cnp <= 9).
// ------------------------------------------------------------------------------------------------
__global__ void mot_solve_kernel(Problem P)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P.m) return;
    const int cnp = P.M.cnp;
    double *da = P.dp + (size_t) j * cnp;
    if (j < P.mcon) {
        for (int ii = 0; ii < cnp; ii++) da[ii] = 0.0;
        return;
    }
    const double mu = *P.mu;
    double L[9][9], y[9];
    const double *Uj = P.U + (size_t) j * cnp * cnp;
    for (int ii = 0; ii < cnp; ii++)
        for (int jj = 0; jj < cnp; jj++) L[ii][jj] = Uj[ii * cnp + jj] + (ii == jj ? mu : 0.0);
    bool ok = true;
    for (int c = 0; c < cnp && ok; c++) {
        double d = L[c][c];
        for (int k = 0; k < c; k++) d -= L[c][k] * L[c][k];
        if (!(d > 0.0)) { ok = false; break; }     // dpotrf: not positive definite
        d = sqrt(d);
        L[c][c] = d;
        for (int r = c + 1; r < cnp; r++) {
            double v = L[r][c];
            for (int k = 0; k < c; k++) v -= L[r][k] * L[c][k];
            L[r][c] = v / d;
        }
    }
    if (!ok) { P.sc->chol_fail = 1; return; }
    const double *ea = P.eab + (size_t) j * cnp;
    for (int r = 0; r < cnp; r++) {
        double v = ea[r];
        for (int k = 0; k < r; k++) v -= L[r][k] * y[k];
        y[r] = v / L[r][r];
    }
    for (int r = cnp - 1; r >= 0; r--) {
        double v = y[r];
        for (int k = r + 1; k < cnp; k++) v -= L[k][r] * da[k];
        da[r] = v / L[r][r];
    }
}

// ------------------------------------------------------------------------------------------------
// K8b: pdp = p + dp, ||dp||^2, dL = sum dp (mu dp + J^T e)   (sba_levmar.c:1443-1447, 1524-1525)
// ------------------------------------------------------------------------------------------------
__global__ void update_kernel(Problem P, const double *p, double *pdp)
{
    cudaGridDependencySynchronize();   // programmatic dependent launch (see launch_pdl)
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const double mu = *P.mu;
    double d2 = 0.0, dl = 0.0;
    if (q < P.nlm) {
        const double d = P.dp[q];
        pdp[q] = p[q] + d;
        d2 = d * d;
        dl = d * (mu * d + P.eab[q]);
    } else if (q < P.nvars) {
        pdp[q] = p[q];      // motion-only BA: the points are not unknowns
    }
    double out;
    if (grid_reduce<0>(d2, P.partial, P.ticket, out)) P.sc->dp_L2 = out;
    if (grid_reduce<0>(dl, P.partial + gridDim.x, P.ticket + 1, out)) P.sc->dL = out;
}

// Wout export (sba_levmar.c:1835-1846): dense (m*cnp) x (3n) matrix, W_ij at rows j*cnp.., columns 3i..
__global__ void wout_scatter_kernel(Problem P, double *Wout)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= P.nvis) return;
    const int cnp = P.M.cnp, j = P.obs_cam[o], i = P.obs_pt[o];
    if (j < P.mcon) return;
    const double *Wo = P.W + (size_t) o * cnp * 3;
    for (int ii = 0; ii < cnp; ii++)
        for (int jj = 0; jj < 3; jj++) Wout[((size_t) j * cnp + ii) * 3 * (size_t) P.n + (size_t) i * 3 + jj] = Wo[ii * 3 + jj];
}

// undamped (V_i)^-1 for the export pass; a singular V_i becomes 100 I (the reference's recovery, sba_levmar.c:1774-1783)
__global__ void vinv_export_kernel(Problem P)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const double *V = P.V + (size_t) i * 9;
    const double a00 = V[0], a01 = V[1], a02 = V[2], a11 = V[4], a12 = V[5], a22 = V[8];
    const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
    const double det = a00 * c00 + a01 * c01 + a02 * c02;
    double *O = P.Vinv + (size_t) i * 9;
    if (!(det != 0.0) || !isfinite(det)) {
        for (int q = 0; q < 9; q++) O[q] = (q % 4 == 0) ? 100.0 : 0.0;
        return;
    }
    const double id = 1.0 / det;
    O[0] = c00 * id; O[1] = c01 * id; O[2] = c02 * id;
    O[3] = c01 * id; O[4] = (a00 * a22 - a02 * a02) * id; O[5] = (a01 * a02 - a00 * a12) * id;
    O[6] = c02 * id; O[7] = O[5]; O[8] = (a00 * a11 - a01 * a01) * id;
}

}  // namespace ba
}  // namespace bsfm
