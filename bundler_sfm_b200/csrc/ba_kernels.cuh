// ba_kernels.cuh -- device data model of the BA hot path (SURVEY.md K1-K8).
//
// All arithmetic is fp64.  Parameter vector p = (a_1..a_m, b_1..b_n): camera j has `cnp` values
// [c(3), w(3), f*f_scale (if est_focal), k1*k_scale, k2*k_scale (if undistort)], point i has 3
// (lib/sfm-driver/sfm.c:652-703).  Observations are stored point-major (the order of `projections`
// / idxij.val, lib/sba-1.5/sba_levmar.c:652-663) with a camera-major permutation beside it.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/bsfm_b200_ba.h"

namespace bsfm {
namespace ba {

constexpr int MAX_CNP = 9;
constexpr int PNP = 3;
constexpr int MNP = 2;
constexpr int SCHUR_CHUNK = 64;        // tuples per partial-sum warp
constexpr int SCHUR_PART_STRIDE = 96;  // doubles per partial (81 block entries + 9 E + pad)

struct Model {
    int cnp, est_focal, undistort, explicit_centers;
    int focal_idx;   // 6 or -1
    int k_idx;       // 7, 6 or -1
    double f_scale, k_scale;
};

// Calibrated camera (camera_params_t::known_intrinsics, K_known, k_known; lib/sfm-driver/sfm.c:339-357): a full
// upper-triangular K and five Brown-Conrady coefficients replace the focal-only pinhole before the radial step.
// Uploaded once per solve, and only when some camera is calibrated.
struct CamIntrinsics {
    double K[5];    // K_known[0], [1], [2], [4], [5] (the reference never reads K_known[3] or [6..8])
    double k[5];    // k_known[0..4]: radial k0, k1, tangential k2, k3, radial k4
    int known;      // known_intrinsics != 0
    int pad;
};

// the table entry of one camera_params_t (host side; solver and outlier pass)
inline CamIntrinsics cam_intrinsics(const bsfm_camera_params_t &c)
{
    CamIntrinsics ci;
    ci.K[0] = c.K_known[0]; ci.K[1] = c.K_known[1]; ci.K[2] = c.K_known[2]; ci.K[3] = c.K_known[4]; ci.K[4] = c.K_known[5];
    for (int q = 0; q < 5; q++) ci.k[q] = c.k_known[q];
    ci.known = c.known_intrinsics ? 1 : 0;
    ci.pad = 0;
    return ci;
}

// Brown-Conrady distortion and K of a calibrated camera (the known_intrinsics branch of sfm_project_rd,
// lib/sfm-driver/sfm.c:339-357), in the reference's operation order
__device__ __forceinline__ void project_known_dev(const CamIntrinsics &ci, double bc0, double bc1, double bc2, double &p0, double &p1)
{
    const double x_n = -bc0 / bc2;
    const double y_n = -bc1 / bc2;
    const double *k = ci.k;
    const double rsq = x_n * x_n + y_n * y_n;
    const double factor = 1.0 + k[0] * rsq + k[1] * rsq * rsq + k[4] * rsq * rsq * rsq;
    const double dx_x = 2.0 * k[2] * x_n * y_n + k[3] * (rsq + 2.0 * x_n * x_n);
    const double dx_y = k[2] * (rsq + 2.0 * y_n * y_n) + 2.0 * k[3] * x_n * y_n;
    const double x_d = x_n * factor + dx_x;
    const double y_d = y_n * factor + dx_y;
    p0 = ci.K[0] * x_d + ci.K[1] * y_d + ci.K[2];
    p1 = ci.K[3] * y_d + ci.K[4];
}

// Fisheye camera (camera_params_t::fisheye, f_cx, f_cy, f_rad, f_angle, f_focal; lib/sfm-driver/sfm.c:426-446): the
// equidistant mapping applied after the pinhole.  Uploaded once per solve, and only when the call asks for the fisheye
// projection (optimize_for_fisheye).
struct CamFisheye {
    double cx, cy, rad, angle, focal;
    int fisheye;    // fisheye != 0
    int pad;
};

inline CamFisheye cam_fisheye(const bsfm_camera_params_t &c)
{
    CamFisheye cf;
    cf.cx = c.f_cx; cf.cy = c.f_cy; cf.rad = c.f_rad; cf.angle = c.f_angle; cf.focal = c.f_focal;
    cf.fisheye = c.fisheye ? 1 : 0;
    cf.pad = 0;
    return cf;
}

constexpr double BSFM_M_PI = 3.14159265358979323846;   // M_PI of the reference's libc headers

// r -> rnew of sfm_fisheye_distort (sfm.c:439-445) in the reference's operation order; r = 0 gives NaN, as there
__device__ __forceinline__ void fisheye_distort_dev(const CamFisheye &cf, double x, double y, double &xd, double &yd)
{
    const double r = sqrt(x * x + y * y);
    const double angle = 180.0 * atan(r / cf.focal) / BSFM_M_PI;
    const double rnew = cf.rad * angle / (0.5 * cf.angle);
    xd = x * (rnew / r) + cf.cx;
    yd = y * (rnew / r) + cf.cy;
}

// scalars produced on the device, copied to pinned host memory once per LM phase
struct Scalars {
    double e_L2;          // sum e^2 of the last residual evaluation
    double dp_L2;         // sum dp^2
    double dL;            // sum dp (mu dp + J^T e)
    double max_pct;       // stop-8 statistic (sba_levmar.c:1552-1561)
    double eab_inf;       // ||J^T e||_inf
    double p_L2;          // sum p^2
    double max_diag;      // max diagonal of U (j >= mcon) and V
    double penalty;       // constraint penalty at p (sba_levmar.c:808-842)
    int singular_v;       // some V*_i could not be inverted
    int chol_fail;        // dense Cholesky hit a non-positive pivot
    int nonfinite;        // residual evaluation produced NaN/Inf
    int pad;
};

struct Problem {
    int n, m, mcon, nvis, nvars, Sdim;
    int nlm;              // LM unknowns: nvars (motion+structure) or m*cnp (motion only, sba_mot_levmar_x: points stay fixed)
    Model M;
    // structure (device)
    const int *rowptr;    // n+1, point-major CRS (idxij.rowptr)
    const int *obs_cam;   // nvis (idxij.colidx)
    const int *obs_pt;    // nvis
    const int *cam_ptr;   // m+1
    const int *cam_obs;   // nvis, observation ids grouped by camera, ascending point
    // Schur structure: upper blocks (j<=k) in ascending (j,k); tuples (obs of j, obs of k) per block
    int nblocks;
    const uint32_t *blk_key;   // j*m + k
    const int *blk_start;      // nblocks+1
    const int4 *tuples;        // (obs_a, obs_b, point, 0)
    int nchunks;
    const int *chunk_off;      // nblocks+1: first chunk of every block
    double *schur_part;        // nchunks * SCHUR_PART_STRIDE
    const int *cam_pos;        // m - mcon: block position of free camera j in S and da (camera_order, ba_order.cu), or null: j - mcon
    // data
    const double *x;       // 2*nvis measurements
    const double *R_init;  // m*9
    const double *f_fixed; // m
    // constraints (device copies; null when unused)
    const char *cam_constrained;    // m*cnp
    const double *cam_constraints;  // m*cnp
    const double *cam_weights;      // m*cnp
    const char *pt_constrained;     // n
    const double *pt_constraints;   // n*3
    const double *pt_weights;       // n
    // work arrays
    double *camR;     // m*4*9 : R(w), R(w + d e_0), R(w + d e_1), R(w + d e_2)
    double *jacA;     // nvis*2*cnp
    double *jacB;     // nvis*6
    double *W;        // nvis*cnp*3
    double *u_part;   // m*nseg*54 partial U/ea sums
    double *U;        // m*cnp*cnp (undamped)
    double *V;        // n*9 (undamped, full symmetric)
    double *Vinv;     // n*9 ((V+mu I)^-1, full symmetric)
    double *eab;      // nvars
    double *S;        // Sdim*Sdim
    double *E;        // Sdim (+ solution workspace)
    double *dp;       // nvars
    double *partial;  // reduction scratch
    unsigned int *ticket;  // last-block counters
    Scalars *sc;      // device scalars
    const double *mu; // damping term of the current try (device scalar, written by the host)
    const CamIntrinsics *intr;  // m entries, or null when no camera is calibrated (then only the KI = false kernels run)
    const CamFisheye *fe;       // m entries, or null without the fisheye projection (then only the FE = false kernels run)
};

// block position of free camera j (>= mcon) in S, E and the dense solution
__device__ __forceinline__ int cam_block(const Problem &P, int j) { return P.cam_pos ? P.cam_pos[j - P.mcon] : j - P.mcon; }

// launch with the programmatic-stream-serialization attribute (PDL): the launch latency of a kernel overlaps
// the tail of its predecessor; every kernel launched this way calls cudaGridDependencySynchronize() before it
// reads anything its predecessors wrote
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// kernels of ba_kernels.cu that the LM solver (ba_solver.cu) launches
__global__ void cam_prep_kernel(Problem P, const double *p, int with_pert);
template <bool KI, bool FE> __global__ void residual_kernel(Problem P, const double *p, double *e_out, const double *e_prev, double eps5);
template <bool KI, bool FE> __global__ void jacobian_kernel(Problem P, const double *p, int jac_mode);
__global__ void v_kernel(Problem P, const double *p, const double *e);
__global__ void u_partial_kernel(Problem P, const double *e, int nseg);
__global__ void u_final_kernel(Problem P, const double *p, int nseg);
__global__ void grad_stats_kernel(Problem P, const double *p);
__global__ void penalty_kernel(Problem P, const double *p);
__global__ void vinv_kernel(Problem P);
__global__ void schur_partial_kernel(Problem P);
__global__ void schur_final_kernel(Problem P);
__global__ void zero_kernel(double *ptr, size_t count);
__global__ void backsub_kernel(Problem P, const double *da);
__global__ void update_kernel(Problem P, const double *p, double *pdp);
__global__ void mot_solve_kernel(Problem P);
__global__ void wout_scatter_kernel(Problem P, double *Wout);
__global__ void vinv_export_kernel(Problem P);

}  // namespace ba
}  // namespace bsfm
