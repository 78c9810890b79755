// ba_outliers.cu -- the reprojection statistics / outlier pass that BundlerApp::RunSFM_SBA runs after every
// run_sfm (src/Bundle.cpp:659-856), on the arguments run_sfm just used (SURVEY.md 8f row 1).
//   per observation : dist = || sfm_project_rd(camera, point) - key ||            (Bundle.cpp:721-754, sfm.c:302-380)
//                     with optimize_for_fisheye, ImageData::DistortPoint after the projection (Bundle.cpp:746-751,
//                     ImageData.cpp:1129-1169)
//   per camera      : med = kth_element_copy(n, iround(0.8 n), dists)             (Bundle.cpp:761-764; qsort.c:152-204:
//                     the k-th smallest, 0.0 when k >= n), thresh = CLAMP(1.2 * 2.0 * med, min, max) (:768-771),
//                     mean and median (iround(0.5 n)) for the log line (:776-788)
//   outliers        : points with dist > thresh in some camera, except protected (constrained) points (:793-823);
//                     the recorded error is the one of the FIRST camera that flags the point (:809-821)
// Compiled with -fmad=false like the other BA kernels: the projection keeps the reference's operation order.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/device/device_segmented_sort.cuh>

#include "common.h"
#include "ba_kernels.cuh"
#include "ba_loop.h"
#include "../../include/bsfm_b200_ba.h"

namespace bsfm {
namespace ba {

// ImageData::DistortPoint (ImageData.cpp:1129-1169) of a fisheye camera, in the reference's operation order: the ray
// (x, y, -f_focal) is rotated by `Rs`; when its z is not positive the point is left as it is (the reference returns
// without writing its aliased output), else it is re-projected and mapped like sfm_fisheye_distort, with
// RAD2DEG(a) = a * (180 / pi) (imagelib/defines.h:32)
__device__ __forceinline__ void distort_point_dev(const CamFisheye &cf, const Rot3 &Rs, double &x, double &y)
{
    const double F = cf.focal;
    const double r0 = Rs.R[0] * x + Rs.R[1] * y + Rs.R[2] * -F;
    const double r1 = Rs.R[3] * x + Rs.R[4] * y + Rs.R[5] * -F;
    const double r2 = Rs.R[6] * x + Rs.R[7] * y + Rs.R[8] * -F;
    if (r2 <= 0.0) return;
    const double xn = r0 * F / r2;
    const double yn = r1 * F / r2;
    const double r = sqrt(xn * xn + yn * yn);
    const double angle = atan(r / F) * (180.0 / BSFM_M_PI);
    const double rnew = cf.rad * angle / (0.5 * cf.angle);
    x = xn * (rnew / r) + cf.cx;
    y = yn * (rnew / r) + cf.cy;
}

// one thread per observation (point-major order == the order of `projections`).  KI: `intr` (m entries) holds the
// calibrated cameras; KI = false never reads it.  FE: `fe` (m entries) holds the fisheye cameras, whose projections
// DistortPoint maps with `Rs`; FE = false never reads them.
template <bool KI, bool FE>
__global__ void outlier_dist_kernel(int nvis, const int *obs_cam, const int *obs_pt, const CamCompact *cams, const CamIntrinsics *intr,
                                    const CamFisheye *fe, Rot3 Rs, const double *pts, const double *proj, int undistort, double *dist)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nvis) return;
    const CamCompact &C = cams[obs_cam[o]];
    const double *b = pts + 3 * (size_t) obs_pt[o];
    // sfm_project_rd with explicit camera centres (Bundle.cpp:741-744 passes `true`), sfm.c:326-338
    const double b0 = b[0] - C.t[0], b1 = b[1] - C.t[1], b2 = b[2] - C.t[2];
    const double c0 = C.R[0] * b0 + C.R[1] * b1 + C.R[2] * b2;
    const double c1 = C.R[3] * b0 + C.R[4] * b1 + C.R[5] * b2;
    const double c2 = C.R[6] * b0 + C.R[7] * b1 + C.R[8] * b2;
    double p0, p1;
    if (KI && intr[obs_cam[o]].known) {
        project_known_dev(intr[obs_cam[o]], c0, c1, c2, p0, p1);
    } else {
        p0 = -c0 * C.f / c2;
        p1 = -c1 * C.f / c2;
    }
    if (undistort) {   // sfm.c:362-377
        const double rsq = (p0 * p0 + p1 * p1) / (C.f * C.f);
        const double factor = 1.0 + C.k0 * rsq + C.k1 * rsq * rsq;
        p0 *= factor;
        p1 *= factor;
    }
    if (FE && fe[obs_cam[o]].fisheye) distort_point_dev(fe[obs_cam[o]], Rs, p0, p1);
    const double dx = p0 - proj[2 * (size_t) o], dy = p1 - proj[2 * (size_t) o + 1];
    dist[o] = sqrt(dx * dx + dy * dy);     // Bundle.cpp:753-756
}

__global__ void outlier_gather_kernel(int count, const int *idx, const double *src, double *dst)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) dst[i] = src[idx[i]];
}

__device__ __forceinline__ int iround_dev(double x) { return (x < 0.0) ? (int) (x - 0.5) : (int) (x + 0.5); }   // util.c:75-81

// one warp per camera: mean (sum in ascending point order), k-th elements from the sorted distances, threshold
__global__ void outlier_cam_stats_kernel(int m, const int *cam_ptr, const double *dist_cam, const double *dist_sorted,
                                         double min_thresh, double max_thresh, double *stats)
{
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (j >= m) return;
    const int s = cam_ptr[j], n = cam_ptr[j + 1] - s;
    double sum = 0.0;
    for (int q = lane; q < n; q += 32) sum += dist_cam[s + q];
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane != 0) return;
    const int k80 = iround_dev(0.8 * n), k50 = iround_dev(0.5 * n);
    const double med80 = (k80 >= n) ? 0.0 : dist_sorted[s + k80];      // kth_element: "k should be < n" -> 0.0 (qsort.c:192-194)
    const double med50 = (k50 >= n) ? 0.0 : dist_sorted[s + k50];
    double thresh = 1.2 * 2.0 * med80;                                   // NUM_STDDEV 2.0 (Bundle.cpp:767-768)
    thresh = (thresh < min_thresh) ? min_thresh : ((thresh > max_thresh) ? max_thresh : thresh);   // CLAMP (defines.h)
    double *o = stats + 5 * (size_t) j;
    o[0] = (double) n; o[1] = sum / n; o[2] = med50; o[3] = med80; o[4] = thresh;
}

// first (lowest-index) camera that flags every point, then that camera's distance
__global__ void outlier_flag_kernel(int nvis, const int *obs_cam, const int *obs_pt, const double *dist, const double *stats,
                                    const char *pt_protected, int *first_cam)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nvis) return;
    const int i = obs_pt[o], j = obs_cam[o];
    if (pt_protected && pt_protected[i]) return;                          // Bundle.cpp:801-806
    if (dist[o] > stats[5 * (size_t) j + 4]) atomicMin(&first_cam[i], j);
}
__global__ void outlier_err_kernel(int nvis, const int *obs_cam, const int *obs_pt, const double *dist, const int *first_cam, double *err)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nvis) return;
    const int i = obs_pt[o];
    if (first_cam[i] == obs_cam[o]) err[i] = dist[o];
}

}  // namespace ba
}  // namespace bsfm

using namespace bsfm;
using namespace bsfm::ba;

// camera tables of a pass (what the loop reads: R, t = centre, f, k; calibrated and fisheye side tables when present)
int bsfm::ba::upload_outlier_cams(const bsfm_camera_params_t *cams, int m, int optimize_for_fisheye, DeviceArena &D, OutlierCams &T)
{
    std::vector<CamCompact> hc(m);
    bool any_known = false;
    for (int j = 0; j < m; j++) {
        memcpy(hc[j].R, cams[j].R, sizeof hc[j].R); memcpy(hc[j].t, cams[j].t, sizeof hc[j].t);
        hc[j].f = cams[j].f; hc[j].k0 = cams[j].k[0]; hc[j].k1 = cams[j].k[1];
        any_known = any_known || cams[j].known_intrinsics;
    }
    TRY(D.upload(&T.cams, hc.data(), (size_t) m));
    if (any_known) {     // calibrated cameras (sfm.c:339-357): side table, only when there is one
        std::vector<CamIntrinsics> hi(m);
        for (int j = 0; j < m; j++) hi[j] = cam_intrinsics(cams[j]);
        TRY(D.upload(&T.intr, hi.data(), (size_t) m));
    }
    if (optimize_for_fisheye) {   // fisheye cameras: side table, only when the call asks for their mapping
        std::vector<CamFisheye> hf(m);
        for (int j = 0; j < m; j++) hf[j] = cam_fisheye(cams[j]);
        TRY(D.upload(&T.fe, hf.data(), (size_t) m));
        // GetRotationFromSpherical(-pi/2, pi/2) (BundleUtil.cpp:70-94), with the host libm like the reference: the identity
        // up to +-6.1e-17 terms, which change the last bits of the result
        const double theta = -0.5 * M_PI, phi = 0.5 * M_PI;
        const double v[3] = {cos(theta) * sin(phi), cos(phi), sin(theta) * sin(phi)};
        const double phi_up = phi - 0.5 * M_PI, theta_up = theta;
        const double up[3] = {cos(theta_up) * sin(phi_up), cos(phi_up), sin(theta_up) * sin(phi_up)};
        const double x_axis[3] = {v[1] * up[2] - v[2] * up[1], v[2] * up[0] - v[0] * up[2], v[0] * up[1] - v[1] * up[0]};
        for (int q = 0; q < 3; q++) { T.Rs.R[q] = x_axis[q]; T.Rs.R[3 + q] = up[q]; T.Rs.R[6 + q] = v[q]; }
    }
    return BSFM_OK;
}

int bsfm::ba::outliers_core(const Visibility &vis, int n, int m, const OutlierCams &T, const double *d_pts, const double *d_proj,
                            int estimate_distortion, double min_thresh, double max_thresh, const char *d_prot, cudaStream_t st,
                            DeviceArena &D, OutlierPass &out)
{
    const int nvis = vis.nvis;
    double *d_dist_cam, *d_dist_sorted;
    TRY(D.alloc(&out.dist, (size_t) nvis)); TRY(D.alloc(&d_dist_cam, (size_t) nvis)); TRY(D.alloc(&d_dist_sorted, (size_t) nvis));
    TRY(D.alloc(&out.stats, (size_t) m * 5)); TRY(D.alloc(&out.err, (size_t) n));
    TRY(D.alloc(&out.first_cam, (size_t) n));
    const int gb = (nvis + 255) / 256;
    const int ud = estimate_distortion ? 1 : 0;
    if (T.fe) {
        if (T.intr) outlier_dist_kernel<true, true><<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, T.cams, T.intr, T.fe, T.Rs, d_pts, d_proj, ud, out.dist);
        else outlier_dist_kernel<false, true><<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, T.cams, nullptr, T.fe, T.Rs, d_pts, d_proj, ud, out.dist);
    } else {
        if (T.intr) outlier_dist_kernel<true, false><<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, T.cams, T.intr, nullptr, T.Rs, d_pts, d_proj, ud, out.dist);
        else outlier_dist_kernel<false, false><<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, T.cams, nullptr, nullptr, T.Rs, d_pts, d_proj, ud, out.dist);
    }
    BSFM_KERNEL_CHECK();

    // per-camera sorted distances, in the camera-major view (ascending point order within each camera)
    outlier_gather_kernel<<<gb, 256, 0, st>>>(nvis, vis.cam_obs, out.dist, d_dist_cam);
    BSFM_KERNEL_CHECK();
    TRY(D.cub(3, [&](void *t, size_t &b) { return cub::DeviceSegmentedSort::SortKeys(t, b, d_dist_cam, d_dist_sorted, nvis, m, vis.cam_ptr, vis.cam_ptr + 1, st); }));
    outlier_cam_stats_kernel<<<(m * 32 + 255) / 256, 256, 0, st>>>(m, vis.cam_ptr, d_dist_cam, d_dist_sorted, min_thresh, max_thresh, out.stats);
    BSFM_KERNEL_CHECK();
    BSFM_CUDA_TRY(cudaMemsetAsync(out.first_cam, 0x7f, (size_t) n * sizeof(int), st));      // 0x7f7f7f7f: larger than any camera index
    outlier_flag_kernel<<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, out.dist, out.stats, d_prot, out.first_cam);
    BSFM_KERNEL_CHECK();
    outlier_err_kernel<<<gb, 256, 0, st>>>(nvis, vis.obs_cam, vis.obs_pt, out.dist, out.first_cam, out.err);
    BSFM_KERNEL_CHECK();
    return BSFM_OK;
}

// the outlier pass on either visibility source (bsfm_reprojection_outliers, bsfm_reprojection_outliers_crs): uploads,
// outliers_core, downloads and the ordering of the list
static int outliers_impl(int num_pts, int num_cameras, const VisSource &vis_src, const double *projections,
                         const bsfm_camera_params_t *cams, const bsfm_v3_t *pts, int estimate_distortion, int fisheye_entry,
                         int optimize_for_fisheye, double min_proj_error_threshold, double max_proj_error_threshold,
                         const char *pt_protected, double *cam_stats, double *obs_dist,
                         int32_t *outliers, double *outlier_errors, int cap, double *global_mean)
{
    clear_error();
    { int rc = require_device(); if (rc != BSFM_OK) return rc; }
    const int n = num_pts, m = num_cameras;
    if (n <= 0 || m <= 0 || !vis_src.present() || !projections || !cams || !pts || cap < 0 || (cap > 0 && (!outliers || !outlier_errors))) {
        set_error("bsfm_reprojection_outliers: bad arguments");
        return BSFM_ERR_ARG;
    }
    for (int j = 0; j < m; j++)
        if (cams[j].fisheye && !fisheye_entry) { set_error("bsfm_reprojection_outliers: fisheye cameras are outside this entry; bsfm_reprojection_outliers_fe takes them"); return BSFM_ERR_UNSUPPORTED; }

    // the legacy default stream, as every copy below: callers may pass device pointers written on it
    DeviceArena D(0);
    Visibility vis;
    TRY(build_visibility(vis_src, n, m, 0, D, vis));
    const int nvis = vis.nvis;
    if (nvis <= 0) { set_error("bsfm_reprojection_outliers: empty visibility mask"); return BSFM_ERR_ARG; }

    OutlierCams T;
    TRY(upload_outlier_cams(cams, m, optimize_for_fisheye, D, T));
    double *d_pts, *d_proj;
    char *d_prot = nullptr;
    TRY(D.upload(&d_pts, pts, (size_t) n * 3));
    TRY(D.upload(&d_proj, projections, (size_t) nvis * 2));
    if (pt_protected) TRY(D.upload(&d_prot, pt_protected, (size_t) n));
    OutlierPass pass;
    TRY(outliers_core(vis, n, m, T, d_pts, d_proj, estimate_distortion, min_proj_error_threshold, max_proj_error_threshold, d_prot, 0, D, pass));
    double *d_dist = pass.dist, *d_stats = pass.stats, *d_err = pass.err;
    int *d_first = pass.first_cam;

    // results
    std::vector<double> stats((size_t) m * 5);
    BSFM_CUDA_TRY(cudaMemcpy(stats.data(), d_stats, stats.size() * sizeof(double), cudaMemcpyDeviceToHost));
    if (cam_stats) memcpy(cam_stats, stats.data(), stats.size() * sizeof(double));
    if (obs_dist) BSFM_CUDA_TRY(cudaMemcpy(obs_dist, d_dist, (size_t) nvis * sizeof(double), cudaMemcpyDefault));
    if (global_mean) {      // Bundle.cpp:790-791, 852-856: sum of the per-camera sums / number of observations
        double tot = 0.0; double cnt = 0.0;
        for (int j = 0; j < m; j++) if (stats[5 * (size_t) j] > 0) { tot += stats[5 * (size_t) j + 1] * stats[5 * (size_t) j]; cnt += stats[5 * (size_t) j]; }
        *global_mean = tot / cnt;
    }
    std::vector<int> first(n);
    std::vector<double> err(n);
    BSFM_CUDA_TRY(cudaMemcpy(first.data(), d_first, (size_t) n * sizeof(int), cudaMemcpyDeviceToHost));
    BSFM_CUDA_TRY(cudaMemcpy(err.data(), d_err, (size_t) n * sizeof(double), cudaMemcpyDeviceToHost));
    std::vector<std::pair<int, int>> found;      // (first flagging camera, point)
    for (int i = 0; i < n; i++) if (first[i] < m) found.push_back(std::make_pair(first[i], i));
    std::sort(found.begin(), found.end());
    const int total = (int) found.size();
    for (int q = 0; q < total && q < cap; q++) { outliers[q] = found[q].second; outlier_errors[q] = err[found[q].second]; }
    return total;
}

extern "C" int bsfm_reprojection_outliers(int num_pts, int num_cameras, const char *vmask, const double *projections,
                                          const bsfm_camera_params_t *cams, const bsfm_v3_t *pts, int estimate_distortion,
                                          double min_proj_error_threshold, double max_proj_error_threshold,
                                          const char *pt_protected, double *cam_stats, double *obs_dist,
                                          int32_t *outliers, double *outlier_errors, int cap, double *global_mean)
{
    return outliers_impl(num_pts, num_cameras, VisSource::mask(vmask), projections, cams, pts, estimate_distortion, 0, 0,
                         min_proj_error_threshold, max_proj_error_threshold, pt_protected, cam_stats, obs_dist, outliers,
                         outlier_errors, cap, global_mean);
}

extern "C" int bsfm_reprojection_outliers_crs(int num_pts, int num_cameras, const int32_t *vis_ptr, const int32_t *vis_cam,
                                              int nvis, const double *projections, const bsfm_camera_params_t *cams,
                                              const bsfm_v3_t *pts, int estimate_distortion,
                                              double min_proj_error_threshold, double max_proj_error_threshold,
                                              const char *pt_protected, double *cam_stats, double *obs_dist,
                                              int32_t *outliers, double *outlier_errors, int cap, double *global_mean)
{
    return outliers_impl(num_pts, num_cameras, VisSource::crs(vis_ptr, vis_cam, nvis), projections, cams, pts,
                         estimate_distortion, 0, 0, min_proj_error_threshold, max_proj_error_threshold, pt_protected, cam_stats,
                         obs_dist, outliers, outlier_errors, cap, global_mean);
}

extern "C" int bsfm_reprojection_outliers_fe(int num_pts, int num_cameras, const char *vmask, const double *projections,
                                             const bsfm_camera_params_t *cams, const bsfm_v3_t *pts, int estimate_distortion,
                                             int optimize_for_fisheye, double min_proj_error_threshold, double max_proj_error_threshold,
                                             const char *pt_protected, double *cam_stats, double *obs_dist,
                                             int32_t *outliers, double *outlier_errors, int cap, double *global_mean)
{
    return outliers_impl(num_pts, num_cameras, VisSource::mask(vmask), projections, cams, pts, estimate_distortion, 1,
                         optimize_for_fisheye, min_proj_error_threshold, max_proj_error_threshold, pt_protected, cam_stats, obs_dist,
                         outliers, outlier_errors, cap, global_mean);
}

extern "C" int bsfm_reprojection_outliers_crs_fe(int num_pts, int num_cameras, const int32_t *vis_ptr, const int32_t *vis_cam,
                                                 int nvis, const double *projections, const bsfm_camera_params_t *cams,
                                                 const bsfm_v3_t *pts, int estimate_distortion, int optimize_for_fisheye,
                                                 double min_proj_error_threshold, double max_proj_error_threshold,
                                                 const char *pt_protected, double *cam_stats, double *obs_dist,
                                                 int32_t *outliers, double *outlier_errors, int cap, double *global_mean)
{
    return outliers_impl(num_pts, num_cameras, VisSource::crs(vis_ptr, vis_cam, nvis), projections, cams, pts,
                         estimate_distortion, 1, optimize_for_fisheye, min_proj_error_threshold, max_proj_error_threshold,
                         pt_protected, cam_stats, obs_dist, outliers, outlier_errors, cap, global_mean);
}
