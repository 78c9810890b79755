/* bsfm_b200_sba.h -- the reference's sba-1.5 driver symbols and the sfm-driver projection callbacks, as exported by the
 * link-time replacements shim/_build/libsba_b200.so and shim/_build/libsfmdrv_b200.so.
 *
 *   sba_motstr_levmar_x   lib/sba-1.5/sba.h:127-138   (expert driver; called by sba_motstr_levmar, sba_levmar_wrap.c:682)
 *   sba_motstr_levmar     lib/sba-1.5/sba.h:96-108    (simple driver; called by run_sfm, lib/sfm-driver/sfm.c:820-838)
 *   sba_mot_levmar(_x)    lib/sba-1.5/sba.h:110-115, :140-145  (motion only; sfm.c:843-856)
 * Signatures are EXACTLY the reference's (tests/c/sba_boundary_main.c is compiled against the reference's own sba.h).
 *
 * A GPU solver cannot call an opaque host callback per observation (SURVEY.md H5), so the callbacks are RECOGNISED:
 *   proj == sfm_project_point3      (sfm.c:503-552)  with adata -> sfm_global_t  ->  bsfm_sba_motstr_levmar_model
 *   proj == sfm_project_point3_mot  (sfm.c:554-561)                              ->  bsfm_sba_mot_levmar_model
 *   proj == sfm_project_point2_fisheye / _mot (sfm.c:448-501, what run_sfm passes with optimize_for_fisheye)
 *                                   -> bsfm_sba_motstr_levmar_model_fe / bsfm_sba_mot_levmar_model_fe with optimize_for_fisheye = 1
 *   expert drivers: func == bsfm_sba_motstr_Qs / bsfm_sba_mot_Qs (the marker the simple drivers of this library pass,
 *   the counterpart of the static sba_motstr_Qs of sba_levmar_wrap.c:73-104) with projac == NULL (finite differences,
 *   what run_sfm uses: sfm.c:821).
 * Anything else -- a foreign projection, an analytic projac, covx != NULL -- fails LOUDLY: message on stderr and
 * SBA_ERROR (-1), the reference's own error convention.  There is no CPU fallback.
 * In the reference these callbacks are `static`; libsfmdrv_b200.so exports them (with a host implementation, so that
 * code which calls them directly keeps working) precisely so that their addresses can be recognised. */
#ifndef BSFM_B200_SBA_H
#define BSFM_B200_SBA_H
#include "bsfm_b200_ba.h"
#ifdef __cplusplus
extern "C" {
#endif

/* == sfm_global_t, lib/sfm-driver/sfm.c:39-54 (field for field; `adata` of the sfm-driver projection callbacks) */
typedef struct {
    int num_cameras, num_points, num_params_per_camera;
    int est_focal_length, const_focal_length, explicit_camera_centers, estimate_distortion;
    bsfm_camera_params_t global_params;
    bsfm_camera_params_t *init_params;
    bsfm_v3_t *points;
} bsfm_sfm_global_t;

/* == sfm_project_point3 / sfm_project_point3_mot (sfm.c:503-561): host evaluation of one projection */
void sfm_project_point3(int j, int i, double *aj, double *bi, double *xij, void *adata);
void sfm_project_point3_mot(int j, int i, double *aj, double *xij, void *adata);
/* == sfm_project_point2_fisheye / sfm_project_point2_fisheye_mot (sfm.c:448-501): host evaluation of one projection */
void sfm_project_point2_fisheye(int j, int i, double *aj, double *bi, double *xij, void *adata);
void sfm_project_point2_fisheye_mot(int j, int i, double *aj, double *xij, void *adata);

struct sba_crsm;
/* markers passed by the simple drivers of libsba_b200 to its expert drivers (never executed by the GPU solver) */
void bsfm_sba_motstr_Qs(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata);
void bsfm_sba_motstr_Qs_fdjac(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata);
void bsfm_sba_mot_Qs(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *hx, void *adata);
void bsfm_sba_mot_Qs_fdjac(double *p, struct sba_crsm *idxij, int *rcidxs, int *rcsubs, double *jac, void *adata);

#ifdef __cplusplus
}
#endif
#endif
