/* shim/sba_b200.c -- link-time drop-in for the reference's libsba.v1.5.a: the four bundle-adjustment drivers with the
 * reference's exact signatures (lib/sba-1.5/sba.h:96-145), forwarding to the GPU solver in libbsfm_b200.so when the
 * projection callback is one it knows.  See include/bsfm_b200_sba.h for the recognition rules and the error behaviour.
 *
 *     gcc -O2 -fPIC -shared -Iinclude shim/sba_b200.c -o libsba_b200.so -L<repo>/bundler_sfm_b200 -lbsfm_b200 -lsfmdrv_b200
 *     ... -o bundler ... -lsfmdrv_b200 -lsba_b200        (instead of -lsfmdrv -lsba.v1.5, src/Makefile:44-45)
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "bsfm_b200_sba.h"

#define SBA_ERROR_RC (-1)

/* == struct wrap_motstr_data_ / wrap_mot_data_ (sba_levmar_wrap.c:30-43): what the simple drivers hand to the expert ones */
struct wrap_motstr { void (*proj)(int, int, double *, double *, double *, void *); void (*projac)(int, int, double *, double *, double *, double *, void *); int cnp, pnp, mnp; void *adata; };
struct wrap_mot { void (*proj)(int, int, double *, double *, void *); void (*projac)(int, int, double *, double *, void *); int cnp, mnp; void *adata; };

static void marker_called(const char *name)
{
    fprintf(stderr, "SBA/b200: %s() is a marker for the GPU solver and evaluates nothing on the host\n", name);
    exit(1);
}
void bsfm_sba_motstr_Qs(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata) { (void) p; (void) idxij; (void) rcidxs; (void) rcsubs; (void) hx; (void) adata; marker_called("bsfm_sba_motstr_Qs"); }
void bsfm_sba_motstr_Qs_fdjac(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata) { (void) p; (void) idxij; (void) rcidxs; (void) rcsubs; (void) jac; (void) adata; marker_called("bsfm_sba_motstr_Qs_fdjac"); }
void bsfm_sba_mot_Qs(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata) { (void) p; (void) idxij; (void) rcidxs; (void) rcsubs; (void) hx; (void) adata; marker_called("bsfm_sba_mot_Qs"); }
void bsfm_sba_mot_Qs_fdjac(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata) { (void) p; (void) idxij; (void) rcidxs; (void) rcsubs; (void) jac; (void) adata; marker_called("bsfm_sba_mot_Qs_fdjac"); }

static int unsupported(const char *fn, const char *what)
{
    fprintf(stderr, "SBA/b200: %s(): %s -- only the sfm-driver projections (sfm_project_point3, sfm_project_point2_fisheye, finite-difference Jacobian, covx == NULL) "
                    "runs on the GPU and there is no CPU fallback\n", fn, what);
    return SBA_ERROR_RC;
}

/* camera model the GPU solver needs, read from the callback's adata (what sfm_project_point3 itself reads, sfm.c:503-552) */
static int model_from_globals(const char *fn, const bsfm_sfm_global_t *g, int m, int cnp, bsfm_sfm_model_t *model, double **R_init, double **f_fixed)
{
    int j;
    if (!g || !g->init_params) return unsupported(fn, "adata is not an sfm_global_t");
    if (g->const_focal_length && g->est_focal_length) return unsupported(fn, "const_focal_length is not implemented (nor in the reference, sfm.c:518-521)");
    if (cnp != 6 + (g->est_focal_length ? 1 : 0) + (g->estimate_distortion ? 2 : 0)) return unsupported(fn, "cnp does not match the sfm camera model");
    *R_init = (double *) malloc((size_t) m * 9 * sizeof(double));
    *f_fixed = (double *) malloc((size_t) m * sizeof(double));
    if (!*R_init || !*f_fixed) { fprintf(stderr, "SBA/b200: %s(): out of memory\n", fn); exit(1); }
    for (j = 0; j < m; j++) {
        if (g->init_params[j].f_scale != g->init_params[0].f_scale || g->init_params[j].k_scale != g->init_params[0].k_scale) {
            free(*R_init); free(*f_fixed); return unsupported(fn, "per-camera f_scale / k_scale differ");
        }
        memcpy(*R_init + (size_t) 9 * j, g->init_params[j].R, 9 * sizeof(double));
        (*f_fixed)[j] = g->init_params[j].f;
    }
    model->est_focal_length = g->est_focal_length; model->undistort = g->estimate_distortion;
    model->explicit_camera_centers = g->explicit_camera_centers;
    model->f_scale = g->init_params[0].f_scale; model->k_scale = g->init_params[0].k_scale;
    model->R_init = *R_init; model->f_fixed = *f_fixed;
    return 0;
}

static int finish(const char *fn, int rc)
{
    if (rc < -1) {      /* BSFM_ERR_*: report like the reference reports its own failures, return SBA_ERROR */
        fprintf(stderr, "SBA/b200: %s() failed: %s\n", fn, bsfm_last_error());
        return SBA_ERROR_RC;
    }
    return rc;
}

/* == sba_motstr_levmar_x, lib/sba-1.5/sba.h:127-138 */
int sba_motstr_levmar_x(const int n, const int m, const int mcon, char *vmask, double *p, const int cnp, const int pnp,
                        double *x, double *covx, const int mnp,
                        void (*func)(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata),
                        void (*fjac)(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata),
                        void *adata, const int itmax, const int verbose, const double *opts /* [SBA_OPTSSZ], 6 entries in the Bundler build */, double *info /* [SBA_INFOSZ] */,
                        int use_constraints, bsfm_camera_constraints_t *constraints,
                        int use_point_constraints, bsfm_point_constraints_t *point_constraints,
                        double *Vout, double *Sout, double *Uout, double *Wout)
{
    static const char fn[] = "sba_motstr_levmar_x";
    const struct wrap_motstr *wd = (const struct wrap_motstr *) adata;
    bsfm_sfm_model_t model;
    double *R_init = NULL, *f_fixed = NULL;
    int rc;
    if (func != bsfm_sba_motstr_Qs || !wd) return unsupported(fn, "unknown `func` callback");
    if (fjac != bsfm_sba_motstr_Qs_fdjac || wd->projac) return unsupported(fn, "analytic Jacobian callback");
    if (wd->proj != sfm_project_point3 && wd->proj != sfm_project_point2_fisheye) return unsupported(fn, "unknown `proj` callback");
    if (covx) return unsupported(fn, "covx != NULL");
    if (wd->cnp != cnp || wd->pnp != pnp || wd->mnp != mnp) return unsupported(fn, "inconsistent block sizes");
    if (itmax == 0) return unsupported(fn, "itmax == 0 (Jacobian verification mode)");
    rc = model_from_globals(fn, (const bsfm_sfm_global_t *) wd->adata, m, cnp, &model, &R_init, &f_fixed);
    if (rc) return rc;
    /* opts really has 6 entries for the Bundler build of sba (it reads opts[5], sba_levmar.c:610) */
    /* calibrated cameras: sfm_project_point3 reads known_intrinsics / K_known / k_known from the same init_params, and
     * sfm_project_point2_fisheye the fisheye fields too */
    rc = bsfm_sba_motstr_levmar_model_fe(n, m, mcon, vmask, p, cnp, pnp, x, NULL, mnp, &model, BSFM_BA_JAC_FD, itmax, verbose, opts, info,
                                         use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout,
                                         ((const bsfm_sfm_global_t *) wd->adata)->init_params, wd->proj == sfm_project_point2_fisheye);
    free(R_init); free(f_fixed);
    return finish(fn, rc);
}

static long count_visible(const char *vmask, long cells)
{
    long i, nvis = 0;
    for (i = 0; i < cells; i++) nvis += (vmask[i] != 0);
    return nvis;
}

/* == sba_motstr_levmar, lib/sba-1.5/sba.h:96-108 / sba_levmar_wrap.c:599-698 */
int sba_motstr_levmar(const int n, const int m, const int mcon, char *vmask, double *p, const int cnp, const int pnp,
                      double *x, double *covx, const int mnp,
                      void (*proj)(int j, int i, double *aj, double *bi, double *xij, void *adata),
                      void (*projac)(int j, int i, double *aj, double *bi, double *Aij, double *Bij, void *adata),
                      void *adata, const int itmax, const int verbose, const double *opts /* [SBA_OPTSSZ], 6 entries in the Bundler build */, double *info /* [SBA_INFOSZ] */,
                      int use_constraints, bsfm_camera_constraints_t *constraints,
                      int use_point_constraints, bsfm_point_constraints_t *point_constraints,
                      double *Vout, double *Sout, double *Uout, double *Wout)
{
    struct wrap_motstr wdata;
    int retval;
    wdata.proj = proj; wdata.projac = projac; wdata.cnp = cnp; wdata.pnp = pnp; wdata.mnp = mnp; wdata.adata = adata;
    if (projac) return unsupported("sba_motstr_levmar", "analytic Jacobian callback");
    retval = sba_motstr_levmar_x(n, m, mcon, vmask, p, cnp, pnp, x, covx, mnp, bsfm_sba_motstr_Qs, bsfm_sba_motstr_Qs_fdjac, &wdata, itmax, verbose,
                                 opts, info, use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout);
    if (info && retval != SBA_ERROR_RC) {     /* each func / fjac evaluation = nvis proj evaluations (sba_levmar_wrap.c:684-695) */
        const long nvis = count_visible(vmask, (long) n * m);
        info[7] *= nvis; info[8] *= nvis;
    }
    return retval;
}

/* == sba_mot_levmar_x, lib/sba-1.5/sba.h:140-145 */
int sba_mot_levmar_x(const int n, const int m, const int mcon, char *vmask, double *p, const int cnp,
                     double *x, double *covx, const int mnp,
                     void (*func)(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata),
                     void (*fjac)(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata),
                     void *adata, const int itmax, const int verbose, const double *opts /* [SBA_OPTSSZ], 6 entries in the Bundler build */, double *info /* [SBA_INFOSZ] */,
                     int use_constraints, bsfm_camera_constraints_t *constraints)
{
    static const char fn[] = "sba_mot_levmar_x";
    const struct wrap_mot *wd = (const struct wrap_mot *) adata;
    const bsfm_sfm_global_t *g;
    bsfm_sfm_model_t model;
    double *R_init = NULL, *f_fixed = NULL;
    int rc;
    if (func != bsfm_sba_mot_Qs || !wd) return unsupported(fn, "unknown `func` callback");
    if (fjac != bsfm_sba_mot_Qs_fdjac || wd->projac) return unsupported(fn, "analytic Jacobian callback");
    if (wd->proj != sfm_project_point3_mot && wd->proj != sfm_project_point2_fisheye_mot) return unsupported(fn, "unknown `proj` callback");
    if (covx) return unsupported(fn, "covx != NULL");
    if (itmax == 0) return unsupported(fn, "itmax == 0 (Jacobian verification mode)");
    g = (const bsfm_sfm_global_t *) wd->adata;
    rc = model_from_globals(fn, g, m, cnp, &model, &R_init, &f_fixed);
    if (rc) return rc;
    if (!g->points) { free(R_init); free(f_fixed); return unsupported(fn, "adata->points is NULL"); }
    rc = bsfm_sba_mot_levmar_model_fe(n, m, mcon, vmask, p, cnp, x, NULL, mnp, &model, (const double *) g->points, BSFM_BA_JAC_FD, itmax, verbose,
                                      opts, info, use_constraints, constraints, g->init_params, wd->proj == sfm_project_point2_fisheye_mot);
    free(R_init); free(f_fixed);
    return finish(fn, rc);
}

/* == sba_mot_levmar, lib/sba-1.5/sba.h:110-115 / sba_levmar_wrap.c:700-780 */
int sba_mot_levmar(const int n, const int m, const int mcon, char *vmask, double *p, const int cnp,
                   double *x, double *covx, const int mnp,
                   void (*proj)(int j, int i, double *aj, double *xij, void *adata),
                   void (*projac)(int j, int i, double *aj, double *Aij, void *adata),
                   void *adata, const int itmax, const int verbose, const double *opts /* [SBA_OPTSSZ], 6 entries in the Bundler build */, double *info /* [SBA_INFOSZ] */,
                   int use_constraints, bsfm_camera_constraints_t *constraints)
{
    struct wrap_mot wdata;
    int retval;
    wdata.proj = proj; wdata.projac = projac; wdata.cnp = cnp; wdata.mnp = mnp; wdata.adata = adata;
    if (projac) return unsupported("sba_mot_levmar", "analytic Jacobian callback");
    retval = sba_mot_levmar_x(n, m, mcon, vmask, p, cnp, x, covx, mnp, bsfm_sba_mot_Qs, bsfm_sba_mot_Qs_fdjac, &wdata, itmax, verbose, opts, info,
                              use_constraints, constraints);
    if (info && retval != SBA_ERROR_RC) {
        const long nvis = count_visible(vmask, (long) n * m);
        info[7] *= nvis; info[8] *= nvis;
    }
    return retval;
}
