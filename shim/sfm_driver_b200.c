/* shim/sfm_driver_b200.c -- link-time drop-in for the reference's libsfmdrv.a (lib/sfm-driver).
 *
 * Exports `run_sfm` with exactly the reference signature (lib/sfm-driver/sfm.h:68-86, extern "C"
 * :23-25) and forwards to bsfm_run_sfm_fe in libbsfm_b200.so (optimize_for_fisheye included).  src/Bundle.cpp (RunSFM_SBA, :645-652)
 * links against this object instead of libsfmdrv.a + libsba.v1.5.a and is otherwise unchanged:
 *
 *     gcc -c shim/sfm_driver_b200.c -Iinclude -o sfm_driver_b200.o
 *     ... -o bundler ... sfm_driver_b200.o -L<repo>/bundler_sfm_b200 -lbsfm_b200   (instead of -lsfmdrv -lsba.v1.5)
 *
 * The struct arguments are layout-identical (include/bsfm_b200_ba.h restates camera_params_t / v3_t).
 * Options the GPU path does not cover (const_focal_length, which the reference does not implement either) terminate like the
 * reference's own fatal paths do (printf + exit(1), sfm.c:56-73): there is deliberately no silent CPU fallback.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "bsfm_b200_sba.h"

void run_sfm(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
             int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
             bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
             int use_constraints, int use_point_constraints, bsfm_v3_t *points_constraints,
             double point_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
             double *Vout, double *Sout, double *Uout, double *Wout)
{
    int rc = bsfm_run_sfm_fe(num_pts, num_cameras, ncons, vmask, projections, est_focal_length, const_focal_length,
                             undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints,
                             use_point_constraints, points_constraints, point_constraint_weight, fix_points,
                             optimize_for_fisheye, eps2, Vout, Sout, Uout, Wout, NULL);
    if (rc < 0) {
        printf("[run_sfm/b200] error %d: %s\n", rc, bsfm_last_error());
        fflush(stdout);
        exit(1);
    }
}

/* ---- the sfm-driver projection callbacks (static in the reference, sfm.c:448-561), exported here so that the sba
 * drop-in (shim/sba_b200.c) can recognise them by address; host evaluation restated from sfm.c:77-116 (rot_update),
 * :302-380 (sfm_project_rd), :243-299 (sfm_project2) and :426-446 (sfm_fisheye_distort) for callers that invoke them
 * directly (the GPU solver never does). ------------------------------------------------------------------------------ */
static void rot_update_host(const double *R, const double *w, double *Rnew)
{
    const double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    double n0, n1, n2, nx[9], nxsq[9], dR[9], sinth, costh;
    int r, c, q;
    if (theta == 0.0) { memcpy(Rnew, R, 9 * sizeof(double)); return; }
    n0 = w[0] / theta; n1 = w[1] / theta; n2 = w[2] / theta;
    nx[0] = 0.0; nx[1] = -n2; nx[2] = n1; nx[3] = n2; nx[4] = 0.0; nx[5] = -n0; nx[6] = -n1; nx[7] = n0; nx[8] = 0.0;
    for (r = 0; r < 3; r++) for (c = 0; c < 3; c++) nxsq[3 * r + c] = nx[3 * r] * nx[c] + nx[3 * r + 1] * nx[3 + c] + nx[3 * r + 2] * nx[6 + c];
    sinth = sin(theta); costh = cos(theta);
    for (q = 0; q < 9; q++) dR[q] = (((q % 4 == 0) ? 1.0 : 0.0) + nx[q] * sinth) + nxsq[q] * (1.0 - costh);
    for (r = 0; r < 3; r++) for (c = 0; c < 3; c++) Rnew[3 * r + c] = dR[3 * r] * R[c] + dR[3 * r + 1] * R[3 + c] + dR[3 * r + 2] * R[6 + c];
}

/* the focal length, rotation update and pinhole of sfm_project_point3 / sfm_project_point2_fisheye (sfm.c:243-299,
 * 339-357, 503-540), before any radial step or fisheye mapping; returns f */
static double project_pinhole(const bsfm_sfm_global_t *g, int j, const double *aj, const double *bi, double *xij)
{
    const bsfm_camera_params_t *init = g->init_params + j;
    const double *dt = aj, *w = aj + 3;
    double f, R[9], b2[3], bc[3];
    if (!g->est_focal_length) f = init->f;
    else if (g->const_focal_length) { printf("Error: case of constant focal length has not been implemented.\n"); f = g->global_params.f; }
    else f = aj[6] / init->f_scale;
    rot_update_host(init->R, w, R);
    if (!g->explicit_camera_centers) {
        bc[0] = R[0] * bi[0] + R[1] * bi[1] + R[2] * bi[2] + dt[0];
        bc[1] = R[3] * bi[0] + R[4] * bi[1] + R[5] * bi[2] + dt[1];
        bc[2] = R[6] * bi[0] + R[7] * bi[1] + R[8] * bi[2] + dt[2];
    } else {
        b2[0] = bi[0] - dt[0]; b2[1] = bi[1] - dt[1]; b2[2] = bi[2] - dt[2];
        bc[0] = R[0] * b2[0] + R[1] * b2[1] + R[2] * b2[2];
        bc[1] = R[3] * b2[0] + R[4] * b2[1] + R[5] * b2[2];
        bc[2] = R[6] * b2[0] + R[7] * b2[1] + R[8] * b2[2];
    }
    if (!init->known_intrinsics) {
        xij[0] = -bc[0] * f / bc[2];
        xij[1] = -bc[1] * f / bc[2];
    } else {    /* calibrated camera: Brown-Conrady k_known, then K_known (sfm.c:339-357) */
        const double *kk = init->k_known, *K = init->K_known;
        const double x_n = -bc[0] / bc[2];
        const double y_n = -bc[1] / bc[2];
        const double rsq = x_n * x_n + y_n * y_n;
        const double factor = 1.0 + kk[0] * rsq + kk[1] * rsq * rsq + kk[4] * rsq * rsq * rsq;
        const double dx_x = 2 * kk[2] * x_n * y_n + kk[3] * (rsq + 2 * x_n * x_n);
        const double dx_y = kk[2] * (rsq + 2 * y_n * y_n) + 2 * kk[3] * x_n * y_n;
        const double x_d = x_n * factor + dx_x;
        const double y_d = y_n * factor + dx_y;
        xij[0] = K[0] * x_d + K[1] * y_d + K[2];
        xij[1] = K[4] * y_d + K[5];
    }
    return f;
}

void sfm_project_point3(int j, int i, double *aj, double *bi, double *xij, void *adata)
{
    const bsfm_sfm_global_t *g = (const bsfm_sfm_global_t *) adata;
    const bsfm_camera_params_t *init = g->init_params + j;
    const double *k = aj + (g->est_focal_length ? 7 : 6);
    const double f = project_pinhole(g, j, aj, bi, xij);
    (void) i;
    if (g->estimate_distortion) {     /* the radial step runs for both kinds of camera and uses f (sfm.c:362-377) */
        const double k1 = k[0] / init->k_scale, k2 = k[1] / init->k_scale;
        const double rsq = (xij[0] * xij[0] + xij[1] * xij[1]) / (f * f);
        const double factor = 1.0 + k1 * rsq + k2 * rsq * rsq;
        xij[0] *= factor; xij[1] *= factor;
    }
}

void sfm_project_point3_mot(int j, int i, double *aj, double *xij, void *adata)
{
    const bsfm_sfm_global_t *g = (const bsfm_sfm_global_t *) adata;
    sfm_project_point3(j, i, aj, g->points[i].p, xij, adata);
}

/* sfm_project_point2_fisheye (sfm.c:448-492): the pinhole without the radial step, then sfm_fisheye_distort (:426-446)
 * for a camera with fisheye != 0; r = 0 gives NaN, as in the reference */
void sfm_project_point2_fisheye(int j, int i, double *aj, double *bi, double *xij, void *adata)
{
    const bsfm_sfm_global_t *g = (const bsfm_sfm_global_t *) adata;
    const bsfm_camera_params_t *cam = g->init_params + j;
    double xn, yn, r, angle, rnew;
    (void) i;
    project_pinhole(g, j, aj, bi, xij);
    if (cam->fisheye == 0) return;
    xn = xij[0]; yn = xij[1];
    r = sqrt(xn * xn + yn * yn);
    angle = 180.0 * atan(r / cam->f_focal) / M_PI;
    rnew = cam->f_rad * angle / (0.5 * cam->f_angle);
    xij[0] = xn * (rnew / r) + cam->f_cx;
    xij[1] = yn * (rnew / r) + cam->f_cy;
}

void sfm_project_point2_fisheye_mot(int j, int i, double *aj, double *xij, void *adata)
{
    const bsfm_sfm_global_t *g = (const bsfm_sfm_global_t *) adata;
    sfm_project_point2_fisheye(j, i, aj, g->points[i].p, xij, adata);
}
