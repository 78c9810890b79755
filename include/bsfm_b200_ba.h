/* bsfm_b200_ba.h -- C ABI of the BA hot path of libbsfm_b200.so (sparse Levenberg-Marquardt bundle
 * adjustment on one H100).  Replaces, behind the reference's own call boundary:
 *
 *   run_sfm(...)                 lib/sfm-driver/sfm.h:68-86,  lib/sfm-driver/sfm.c:592-1003
 *   sba_motstr_levmar_x(...)     lib/sba-1.5/sba.h:127-138,   lib/sba-1.5/sba_levmar.c:457-2081
 *
 * The structs below restate the reference's interface types field-for-field so that a caller
 * compiled against the reference headers can pass its own objects unchanged (same size, same
 * offsets; checked by tests/test_abi.py against the compiled reference when it is available).
 * There is no CPU fallback; unsupported reference options return BSFM_ERR_UNSUPPORTED.
 */
#ifndef BSFM_B200_BA_H
#define BSFM_B200_BA_H

#include <stdint.h>
#include "bsfm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BSFM_NUM_CAMERA_PARAMS 9     /* lib/sfm-driver/sfm.h:29 */
#define BSFM_POLY_INVERSE_DEGREE 6   /* lib/sfm-driver/sfm.h:30 */

/* == camera_params_t, lib/sfm-driver/sfm.h:32-51 */
typedef struct {
    double R[9];
    double t[3];
    double f;
    double k[2];
    double k_inv[BSFM_POLY_INVERSE_DEGREE];
    char constrained[BSFM_NUM_CAMERA_PARAMS];
    double constraints[BSFM_NUM_CAMERA_PARAMS];
    double weights[BSFM_NUM_CAMERA_PARAMS];
    double K_known[9];
    double k_known[5];
    char fisheye;
    char known_intrinsics;
    double f_cx, f_cy;
    double f_rad, f_angle;
    double f_focal;
    double f_scale, k_scale;
} bsfm_camera_params_t;

/* == v3_t, lib/matrix/vector.h:65-67 */
typedef struct { double p[3]; } bsfm_v3_t;

/* == camera_constraints_t / point_constraints_t, lib/sba-1.5/sba.h:80-90 */
typedef struct { char *constrained; double *constraints; double *weights; } bsfm_camera_constraints_t;
typedef struct { char constrained; double constraints[3]; double weight; } bsfm_point_constraints_t;

/* Jacobian mode of the solver (env BSFM_BA_JAC overrides: "fd" | "analytic")
 *   0 = forward finite differences with the reference's step rule d = max(1e-4*|p|, 1e-6)
 *       (lib/sba-1.5/sba_levmar_wrap.c:203-256, sba.h:52-53) -- what run_sfm uses (projac = NULL,
 *       lib/sfm-driver/sfm.c:820-828); the parity mode and the default.
 *   1 = analytic 2x9 / 2x3 Jacobians of the same camera model (include/snavely_reprojection_error.h:58-92
 *       restated in the SBA parameterisation, SURVEY.md Appendix A.4)                            */
#define BSFM_BA_JAC_FD        0
#define BSFM_BA_JAC_ANALYTIC  1

/* Camera model descriptor: what sfm_project_point3 (lib/sfm-driver/sfm.c:503-552) reads from its
 * `adata` (sfm_global_t) -- made explicit because a GPU solver cannot call an opaque callback.   */
typedef struct {
    int est_focal_length;         /* aj[6] = f * f_scale is a parameter (else f_fixed[j] is used)   */
    int undistort;                /* two radial terms k1,k2 (scaled by k_scale) are parameters       */
    int explicit_camera_centers;  /* aj[0..2] is the camera centre c (P = R (X - c)), else P = R X + t */
    double f_scale, k_scale;      /* 0.001 and 5.0 in run_sfm (sfm.c:634-635)                        */
    const double *R_init;         /* m x 9 row-major initial rotations (init_params[j].R)            */
    const double *f_fixed;        /* m focal lengths used when est_focal_length == 0                 */
} bsfm_sfm_model_t;

/* Core solver == sba_motstr_levmar_x (lib/sba-1.5/sba_levmar.c:457-2081) with func/fjac/adata
 * replaced by the explicit camera model.  Arguments keep the reference's meaning:
 *   n points, m cameras, mcon leading cameras held fixed, vmask n x m, p = (a_1..a_m, b_1..b_n)
 *   in/out, cnp in {6,7,8,9}, pnp = 3, x = measurements (2 per visible projection, point-major),
 *   covx must be NULL, mnp = 2, itmax, verbose, opts[6] (reads opts[5], sba_levmar.c:610),
 *   info[10] (sba_levmar.c:2028-2049), camera / point constraints as in sba.h:80-90.
 * vmask, p and x may be host pointers or device pointers (unified addressing decides the copy kind);
 * with device pointers no bulk host<->device copy happens inside the call (bench `value` leg).
 * Vout/Sout/Uout/Wout (nullable) export the undamped V (n x 9), reduced camera matrix S ((m cnp)^2), U (m x cnp^2)
 * and W (dense (m cnp) x (3n)) like sba_levmar.c:1633-2026 (extra Jacobian + Schur pass when Sout != NULL; mcon == 0).
 * Returns the number of iterations (>=0) like the reference, SBA_ERROR (-1) where the reference
 * returns it, or another negative BSFM_ERR_* code.                                              */
int bsfm_sba_motstr_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                 const double *x, const double *covx, int mnp,
                                 const bsfm_sfm_model_t *model, int jac_mode,
                                 int itmax, int verbose, const double opts[6], double info[10],
                                 int use_constraints, const bsfm_camera_constraints_t *constraints,
                                 int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                 double *Vout, double *Sout, double *Uout, double *Wout);

/* Motion-only solver == sba_mot_levmar_x (lib/sba-1.5/sba.h:157-166, lib/sba-1.5/sba_levmar.c:2090-2690) with
 * func/fjac/adata replaced by the explicit camera model: only the cameras are unknowns, the n points are read from
 * `points` (n x 3, host or device; what sfm_project_point3_mot takes from its adata, lib/sfm-driver/sfm.c:553-560)
 * and never change.  p = (a_1..a_m) in/out.  The augmented normal equations are block diagonal,
 * (U_j + mu I) da_j = ea_j per camera (sba_levmar.c:2487-2514).  The LM controller is the stock SBA one: it has no
 * stop-8 rule and prints no max_pct_change; info[9] counts one linear system per camera and try (:2513).
 * Returns like bsfm_sba_motstr_levmar_model.                                                                    */
int bsfm_sba_mot_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                              const double *x, const double *covx, int mnp,
                              const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                              int itmax, int verbose, const double opts[6], double info[10],
                              int use_constraints, const bsfm_camera_constraints_t *constraints);

/* The two solvers above with calibrated cameras.  init_params (nullable, m entries) is what sfm_project_point3 reads
 * from its adata besides the model: a camera with known_intrinsics != 0 projects through its own K_known[0,1,2,4,5]
 * and Brown-Conrady k_known[0..4] instead of the focal-only pinhole (lib/sfm-driver/sfm.c:339-357), followed by the
 * same optional radial step, which still uses the focal parameter (aj[6] / f_scale or f_fixed[j]) and aj's k1, k2.
 * Only known_intrinsics, K_known and k_known are read; cameras may be mixed.  Unlike vmask, p and x, init_params is
 * read on the host during setup and must be host memory.  With init_params == NULL, or with no
 * calibrated camera in it, these are exactly bsfm_sba_motstr_levmar_model / bsfm_sba_mot_levmar_model, which call
 * them with NULL.  Both Jacobian modes cover calibrated cameras.                                                 */
int bsfm_sba_motstr_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                    const double *x, const double *covx, int mnp,
                                    const bsfm_sfm_model_t *model, int jac_mode,
                                    int itmax, int verbose, const double opts[6], double info[10],
                                    int use_constraints, const bsfm_camera_constraints_t *constraints,
                                    int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                    double *Vout, double *Sout, double *Uout, double *Wout,
                                    const bsfm_camera_params_t *init_params);
int bsfm_sba_mot_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                 const double *x, const double *covx, int mnp,
                                 const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                 int itmax, int verbose, const double opts[6], double info[10],
                                 int use_constraints, const bsfm_camera_constraints_t *constraints,
                                 const bsfm_camera_params_t *init_params);

/* The two _ki solvers above with the fisheye projection of run_sfm's optimize_for_fisheye (sfm_project_point2_fisheye
 * and its _mot twin, lib/sfm-driver/sfm.c:448-501).  optimize_for_fisheye == 0: exactly the _ki entries.  With 1, every
 * camera projects through the pinhole (focal-only, or K_known / k_known for a calibrated camera) WITHOUT the radial step,
 * so with undistort the k1, k2 columns of the Jacobian are exactly zero and only camera constraints move them; then a
 * camera with fisheye != 0 maps the pinhole point u to u * rnew / |u| + (f_cx, f_cy), rnew = f_rad * angle / (f_angle / 2),
 * angle = 180 atan(|u| / f_focal) / pi (sfm_fisheye_distort, :426-446).  A point on a fisheye camera's principal axis
 * gives NaN, as in the reference (it ends the solve through stop 7).  init_params (host memory) is required with 1; its
 * fisheye, f_cx, f_cy, f_rad, f_angle, f_focal fields are read besides the calibration.  Both Jacobian modes cover it. */
int bsfm_sba_motstr_levmar_model_fe(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                    const double *x, const double *covx, int mnp,
                                    const bsfm_sfm_model_t *model, int jac_mode,
                                    int itmax, int verbose, const double opts[6], double info[10],
                                    int use_constraints, const bsfm_camera_constraints_t *constraints,
                                    int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                    double *Vout, double *Sout, double *Uout, double *Wout,
                                    const bsfm_camera_params_t *init_params, int optimize_for_fisheye);
int bsfm_sba_mot_levmar_model_fe(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                 const double *x, const double *covx, int mnp,
                                 const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                 int itmax, int verbose, const double opts[6], double info[10],
                                 int use_constraints, const bsfm_camera_constraints_t *constraints,
                                 const bsfm_camera_params_t *init_params, int optimize_for_fisheye);

/* == run_sfm (lib/sfm-driver/sfm.h:68-86): same arguments, same in/out semantics
 * (init_camera_params and init_pts are overwritten with the solution, sfm.c:876-929; prints
 * "[run_sfm] Number of iterations" / "info[6]" like sfm.c:872-873), plus `info_out` (nullable,
 * 10 doubles) and an int return (0 or negative error) which the void reference lacks.
 * fix_points == 1 runs the motion-only solver (sfm.c:843-849; init_pts untouched).  Cameras with
 * known_intrinsics != 0 project through their K_known / k_known (see bsfm_sba_motstr_levmar_model_ki), which
 * run_sfm neither packs nor changes.  This entry covers optimize_for_fisheye == 0 and const_focal_length == 0;
 * anything else returns BSFM_ERR_UNSUPPORTED (callers may rely on that to route fisheye work elsewhere);
 * bsfm_run_sfm_fe runs optimize_for_fisheye == 1.                                              */
int bsfm_run_sfm(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
                 int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                 bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                 int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
                 double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                 double *Vout, double *Sout, double *Uout, double *Wout, double *info_out);

/* Visibility in CRS form, accepted by the _crs entries below in place of the dense num_pts x num_cameras vmask.  It is
 * the layout sba builds from vmask itself (idxij, lib/sba-1.5/sba_levmar.c:652-663):
 *   vis_ptr (num_pts + 1): point i's observations are [vis_ptr[i], vis_ptr[i + 1])
 *   vis_cam (nvis):        the camera of each observation, strictly ascending within a point
 * `projections` keep the order of the dense entries: point-major, ascending camera within a point, i.e. observation q
 * of the CRS.  vis_ptr and vis_cam may be host (pageable or pinned) or device pointers, like vmask.  A vmask and the CRS
 * of its non-zero bytes give bitwise identical results.  The arrays are checked on the device before anything reads
 * them; the call returns BSFM_ERR_ARG, with a message naming the lowest offending point and the fault, when
 *   nvis < 0 or 2 * nvis overflows int;  vis_ptr[0] != 0 (point 0);  vis_ptr[num_pts] != nvis (point num_pts - 1);
 *   vis_ptr[i] or vis_ptr[i + 1] outside [0, nvis], or vis_ptr[i + 1] < vis_ptr[i] (point i);
 *   a camera index outside [0, num_cameras), or cameras not strictly ascending, in point i's observations.
 * For one point the faults are reported in this order.  vis_cam may be NULL when nvis == 0.                          */

/* bsfm_run_sfm (run_sfm, lib/sfm-driver/sfm.c:592-1003) with the visibility as CRS: every other argument, return code,
 * print and in/out rule is that of bsfm_run_sfm.  nvis == 0 returns SBA_ERROR (-1), "fewer measurements than
 * unknowns", like an empty vmask.                                                                                 */
int bsfm_run_sfm_crs(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                     double *projections, int est_focal_length, int const_focal_length, int undistort,
                     int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                     int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
                     double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                     double *Vout, double *Sout, double *Uout, double *Wout, double *info_out);

/* bsfm_run_sfm and bsfm_run_sfm_crs, same arguments, honouring optimize_for_fisheye: with 1 the solver projects like
 * sfm_project_point2_fisheye (see bsfm_sba_motstr_levmar_model_fe; fix_points selects the _mot twin, sfm.c:829-856),
 * reading each camera's fisheye fields from init_camera_params, which it leaves as they are.  With 0 these are
 * bit-identical to the entries they extend, fisheye cameras included (their fisheye byte is not read then).        */
int bsfm_run_sfm_fe(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
                    int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                    bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                    int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
                    double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                    double *Vout, double *Sout, double *Uout, double *Wout, double *info_out);
int bsfm_run_sfm_crs_fe(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                        double *projections, int est_focal_length, int const_focal_length, int undistort,
                        int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                        int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
                        double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                        double *Vout, double *Sout, double *Uout, double *Wout, double *info_out);

/* The reprojection statistics / outlier pass BundlerApp::RunSFM_SBA runs after every run_sfm on the same
 * vmask / projections / cameras / points (src/Bundle.cpp:659-856), as one call (SURVEY.md 8f row 1):
 *   dist(obs)   = || sfm_project_rd(camera, point, estimate_distortion, explicit centres) - measurement ||  (:721-754)
 *   per camera  : med80 = kth_element_copy(n, iround(0.8 n), dists) (0.0 when that index is >= n, lib/imagelib/
 *                 qsort.c:191-194), thresh = CLAMP(1.2 * 2.0 * med80, min_thresh, max_thresh)  (:761-771)
 *   outliers    : every point with dist > thresh in some camera, unless pt_protected[point] != 0 (the caller's
 *                 "constrained point" rule, :801-806); the reported error is the distance in the first (lowest
 *                 index) camera that flags the point, like the reference's first-found rule (:809-821)
 * cameras: the `R`, `t` (= centre), `f`, `k` fields of run_sfm's output are read, and for cameras with known_intrinsics
 *   != 0 also K_known and k_known (sfm.c:339-357, then the radial step with f and k).  fisheye cameras are refused
 *   (bsfm_reprojection_outliers_fe takes them).
 * cam_stats (nullable): num_cameras x 5 = { #observations, mean distance, median (iround(0.5 n)-th), med80, thresh }
 * obs_dist  (nullable): one distance per observation in the order of `projections`
 * outliers / outlier_errors: up to `cap` entries, ordered by (first flagging camera, point index) -- the
 *   reference lists them by (camera, key index); same set, same errors
 * global_mean (nullable): the "[RunSFM] Global mean reprojection error" value (:852-856)
 * Returns the number of outliers (may exceed cap) or a negative error.  Host or device pointers for vmask,
 * projections, pts.                                                                                          */
int bsfm_reprojection_outliers(int num_pts, int num_cameras, const char *vmask, const double *projections,
                               const bsfm_camera_params_t *cams, const bsfm_v3_t *pts, int estimate_distortion,
                               double min_proj_error_threshold, double max_proj_error_threshold,
                               const char *pt_protected, double *cam_stats, double *obs_dist,
                               int32_t *outliers, double *outlier_errors, int cap, double *global_mean);

/* bsfm_reprojection_outliers (src/Bundle.cpp:659-856) with the visibility as CRS (see bsfm_run_sfm_crs): every other
 * argument and output is that of bsfm_reprojection_outliers.  nvis == 0 returns BSFM_ERR_ARG, "empty visibility",
 * like an empty vmask.                                                                                           */
int bsfm_reprojection_outliers_crs(int num_pts, int num_cameras, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                                   const double *projections, const bsfm_camera_params_t *cams, const bsfm_v3_t *pts,
                                   int estimate_distortion, double min_proj_error_threshold, double max_proj_error_threshold,
                                   const char *pt_protected, double *cam_stats, double *obs_dist,
                                   int32_t *outliers, double *outlier_errors, int cap, double *global_mean);

/* The two outlier entries above with an optimize_for_fisheye argument after estimate_distortion; they accept fisheye
 * cameras either way, as the reference does.  With 1, a camera with fisheye != 0 passes its sfm_project_rd projection
 * through ImageData::DistortPoint (src/Bundle.cpp:746-751, ImageData.cpp:1129-1169): the ray (x, y, -f_focal), rotated
 * by GetRotationFromSpherical(-pi/2, pi/2) (computed on the host with the C library's cos / sin), is re-projected and
 * mapped like sfm_fisheye_distort with RAD2DEG(a) = a * (180 / pi); a ray whose rotated z is <= 0 keeps the undistorted
 * projection.  With 0 every camera is projected as an ordinary (or calibrated) one.                                   */
int bsfm_reprojection_outliers_fe(int num_pts, int num_cameras, const char *vmask, const double *projections,
                                  const bsfm_camera_params_t *cams, const bsfm_v3_t *pts, int estimate_distortion,
                                  int optimize_for_fisheye, double min_proj_error_threshold, double max_proj_error_threshold,
                                  const char *pt_protected, double *cam_stats, double *obs_dist,
                                  int32_t *outliers, double *outlier_errors, int cap, double *global_mean);
int bsfm_reprojection_outliers_crs_fe(int num_pts, int num_cameras, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                                      const double *projections, const bsfm_camera_params_t *cams, const bsfm_v3_t *pts,
                                      int estimate_distortion, int optimize_for_fisheye,
                                      double min_proj_error_threshold, double max_proj_error_threshold,
                                      const char *pt_protected, double *cam_stats, double *obs_dist,
                                      int32_t *outliers, double *outlier_errors, int cap, double *global_mean);

/* One round of bsfm_run_sfm_outlier_loop */
typedef struct {
    int32_t num_pts;        /* points solved this round (the reference's nz_count, src/Bundle.cpp:613-637) */
    int32_t nvis;           /* observations solved this round */
    int32_t num_outliers;   /* points flagged by this round's outlier pass */
    int32_t removed;        /* 1 when they were removed (remove_outliers != 0) */
    double  info[10];       /* sba's info[] of this round's solve */
    double  global_mean;    /* "[RunSFM] Global mean reprojection error" of this round (:852-856) */
    int64_t h2d_bytes;      /* bytes the round's setup (scene, cameras, tables, structure) copied from host to device ... */
    int64_t h2d_largest;    /* ... and its largest single copy.  Round 0 includes the upload of the scene; the 8-byte */
                            /* damping term the controller sends per LM try is not counted. */
} bsfm_sfm_round_t;

/* The solve / outlier-removal loop of BundlerApp::RunSFM_SBA (src/Bundle.cpp:568-919) as one call: bsfm_run_sfm_crs_fe,
 * bsfm_reprojection_outliers_crs_fe and the removal of the flagged points, repeated until a round flags at most
 * min_outliers points.  The scene is uploaded once and stays on the device between rounds; a round is bit-identical to
 * the two separate calls on the same inputs.  After the first round the host sends only the cameras (packed parameters and
 * the tables the kernels read) and reads back the cameras, the per-camera statistics and three counts.
 *   visibility   CRS only (see bsfm_run_sfm_crs; host or device pointers), checked once with the same BSFM_ERR_ARG
 *                messages.  RunSFM_SBA holds tracks (pt_views); the dense mask it builds from them every round
 *                (:606-623) is the cost this entry avoids.
 *   dropping     before every round, points without views leave the problem and the others are renumbered densely in
 *                ascending original index (remap, :614-636) -- on entry too (pt_round = -2).  init_pts[i] of a point that
 *                was dropped keeps the value it had when it was last solved (:905-909).
 *   loop control at the top of every round, num_pts - (outliers removed so far) < min_points, on the ORIGINAL num_pts,
 *                prints "[RunSFM] Too few points remaining, exiting!" and ends the loop with *mean_error = DBL_MAX
 *                (:588-595).  Otherwise the loop runs while the last round removed more than min_outliers points (:913);
 *                a round that flags fewer still removes them, then stops.  remove_outliers == 0 runs exactly one round and
 *                removes nothing (:858, :911).  Bundler's values: min_outliers 40, min_points 20.
 *   protection   a point with use_point_constraints && points_constraints[i].p[0] != 0.0, i its ORIGINAL index, is never
 *                flagged (:800-806).
 *   QUIRK        the reference hands m_point_constraints to run_sfm as it is (:651), so the SOLVE reads
 *                points_constraints[q] for the index q a point has in that round (sfm.c:757-781), while the protection
 *                test reads the original index.  Once a point below a constrained one has been removed (or had no view on
 *                entry) the two disagree: the constraint then pulls on the point that took the constrained point's place.
 *                This entry does what the reference does; points_constraints is never compacted.
 *   outliers     whole points: all views of a flagged point go away (:871-889).  Flagging, thresholds, the reported error
 *                (first flagging camera) and the fisheye DistortPoint step are those of bsfm_reprojection_outliers_crs_fe
 *                with estimate_distortion = undistort (:647, :739).
 *   solver       fix_points = 1 runs the motion-only solver every round; optimize_for_fisheye is honoured;
 *                const_focal_length is refused as in bsfm_run_sfm.  V/S/U/W are not exported: Bundler asks for them only
 *                on the two-camera first solve (src/Bundle.cpp:2150-2154), which goes to bsfm_run_sfm.  k_inv
 *                (InvertDistortion, :680-705) needs image sizes and stays with the caller.  A solve that ends with
 *                SBA_ERROR continues to the outlier pass, like run_sfm.
 *   prints       per round the two lines of bsfm_run_sfm, and the too-few-points line.
 * Outputs: init_camera_params, init_pts (in/out, by original index); pt_round[num_pts] = the round (0-based) whose pass
 * removed the point, -1 kept, -2 no view on entry; pt_error[num_pts] = the reported reprojection error of a removed point
 * (0 otherwise); cam_stats (nullable, num_cameras x 5, layout of bsfm_reprojection_outliers) of the LAST round;
 * rounds[min(rounds_cap, return value)]; *mean_error = RunSFM_SBA's return value, the mean distance over the observations
 * of the last round (its global_mean; the reference adds the same distances in one running sum), 0 when no round ran.
 * Returns the number of rounds run (>= 0, may exceed rounds_cap) or a negative BSFM_ERR_*; then the outputs hold what
 * the completed rounds left.                                                                                          */
int bsfm_run_sfm_outlier_loop(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                              const double *projections, int est_focal_length, int const_focal_length, int undistort,
                              int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                              int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
                              double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                              int remove_outliers, int min_outliers, int min_points,
                              double min_proj_error_threshold, double max_proj_error_threshold,
                              int32_t *pt_round, double *pt_error, double *cam_stats,
                              bsfm_sfm_round_t *rounds, int rounds_cap, double *mean_error);

/* == sba_Axb_Chol (lib/sba-1.5/sba_lapack.c:374-485, called at sba_levmar.c:1343): x = A^-1 B for a symmetric
 * positive definite m x m matrix (dpotrf + dpotrs in the reference).  A, B, x: host or device pointers; A and B are
 * NOT modified (the reference overwrites them when iscolmaj == 1).  Returns 1 on success, 0 when A is not positive
 * definite -- the reference's own return values -- and a negative BSFM_ERR_* on a library error.
 * Systems above 1536 unknowns run the 256-column panel factorisation whose trailing update runs on the fp64 tensor
 * cores (csrc/ba_chol_large.cu); smaller ones the latency-optimised path (csrc/ba_chol.cu).                          */
int bsfm_sba_Axb_Chol(const double *A, const double *B, double *x, int m, int iscolmaj);
/* the same solve repeated `reps` times on a fresh copy of A; *ms_per_solve = mean device time (CUDA events) of one
 * factorisation + both triangular solves (measurement entry used by bench.py and the tests)                          */
int bsfm_sba_Axb_Chol_timed(const double *A, const double *B, double *x, int m, int reps, float *ms_per_solve);
/* Test / diagnostic entry: the solve of bsfm_sba_Axb_Chol (same launches, same return values and x), plus what it
 * computed on the way.  Every output may be NULL; all are copied out even when the factorisation fails.
 *   L          m x m row-major: the lower triangle of the factor.  Every path writes only that triangle of a zeroed
 *              matrix, so the upper part comes back as +0.
 *   linv       ceil(m/32) blocks of 32 x 32 row-major, block k = (L_kk)^-1 of the k-th diagonal 32-block (lower
 *              triangular, zero above the diagonal), written by chol_step_kernel (m <= 32 and 641..1536), the
 *              dataflow kernel (33..640 and the last panels of larger systems) or chol_diag_kernel (the other panels of
 *              m > 1536).  In a partial last block only rows and columns < m mod 32 are the inverse.
 *   xinv       m > 1536 only (ignored otherwise): ceil(m/256) blocks of 256 x 256 row-major, block p = (L_pp)^-T of the
 *              p-th diagonal 256-block (upper triangular), which the back substitution multiplies with.  In a partial
 *              last block only rows and columns < m mod 256 are written.
 *   fail_code  the raw failure word of the factorisation: 0 none, 1 a non-positive or non-finite pivot, 2 a word of the
 *              dataflow kernel (csrc/ba_chol_dataflow.cu) that never arrived.  Any nonzero value returns 0.       */
int bsfm_sba_Axb_Chol_factor(const double *A, const double *B, double *x, int m, double *L, double *linv, double *xinv,
                             int *fail_code);
/* Test entry: bsfm_sba_Axb_Chol_factor on a matrix with the caller's row envelope: first_col[i] (0 <= first_col[i] <= i)
 * is the first nonzero column of row i, and entries of A left of it are taken as zero.  For m > 4096 whose band plan fits
 * (bsfm_ba_chol_band_plan with the device's SM count - 1 workers) the one-launch band factorisation runs; L is then written
 * on the envelope's 32 x 32 tiles only, and xinv is not written.  Otherwise the same solve as bsfm_sba_Axb_Chol_factor.   */
int bsfm_sba_Axb_Chol_factor_env(const double *A, const double *B, double *x, int m, const int32_t *first_col, double *L,
                                 double *linv, double *xinv, int *fail_code);
/* The band plan of an n x n system with row envelope first_col (host only): env (may be NULL; ceil(n/32) + 1 entries)
 * receives the first tile column of every 32-row block (the right-hand-side row last, 0); out[0] = tiles of the envelope,
 * right-hand-side row included, out[1] = the largest number of tiles taking updates at one step, out[2] = worker CTAs the
 * schedule uses (0 when it does not fit).  Returns 1 when 4096 < n <= 24576 and the plan fits `workers` CTAs of two tile
 * slots each and the solver's workspace, 0 when not, < 0 on bad arguments.  Smaller systems keep the panel path.                                                                 */
int bsfm_ba_chol_band_plan(int n, const int32_t *first_col, int workers, int32_t *env, int64_t out[3]);

/* Per-kernel-class device timing of the large-system Cholesky (systems > 1536 unknowns), for roofline reporting:
 * bsfm_ba_chol_profile(1) resets the counters of the calling thread and records CUDA events around every launch of
 * the following solves; bsfm_ba_chol_profile_read returns accumulated ms / launch counts for
 * [0] diagonal-block factorisation  [1] panel solve  [2] trailing update  [3] back substitution,
 * and the fp64 FLOPs of the trailing update (2 per multiply-add of the lower triangle).  Call it after the solves
 * have completed.  [0] includes the diagonal blocks the look-ahead factors on its side stream, next to the trailing update
 * (their time overlaps [2]).  On the band path (a banded system whose plan fits) the one factorisation launch counts in
 * [0], its back substitution in [3], and [1], [2] and the FLOPs stay 0.                                              */
int bsfm_ba_chol_profile(int enable);
int bsfm_ba_chol_profile_read(float ms[4], int launches[4], double *fp64_flops);

/* Camera order of a motion+structure solve whose reduced camera system takes the large Cholesky path
 * ((m - mcon) * cnp > 1536 unknowns); host only.  blk_key[0 .. nblocks): the Schur blocks j * m + k (j <= k; cameras
 * j, k >= mcon share a point; diagonal keys may be present).  Scores the natural camera order and reverse Cuthill-McKee
 * by the 128 x 128 tiles the trailing update keeps over the whole factorisation (scores[0] natural, scores[1] RCM), from
 * the symbolic block structure of the factor, and takes RCM when it keeps at most 3/4 of the natural order's tiles.
 * cam_pos[j - mcon] receives the block position of free camera j (m - mcon entries; the identity when the natural order
 * is kept).  Smaller systems keep the natural order, unscored (scores 0).  Returns 1 for RCM, 0 for the natural order,
 * < 0 on bad arguments.  The solver applies the order unless BSFM_BA_CAMERA_ORDER=0.                                   */
int bsfm_ba_camera_order(int m, int mcon, int cnp, const uint32_t *blk_key, int nblocks, int32_t *cam_pos, int64_t scores[2]);

/* Per-phase device time (ms, CUDA events) of the last solve of this thread:
 * [0] setup (H2D, CSR, Schur structure)  [1] residual/Jacobian/U/V/W  [2] Schur S assembly
 * [3] dense Cholesky + solves  [4] back-substitution/update/function eval  [5] whole solve      */
int bsfm_ba_last_timing(float ms[6], int *iterations, int *launches);

#ifdef __cplusplus
}
#endif
#endif /* BSFM_B200_BA_H */
