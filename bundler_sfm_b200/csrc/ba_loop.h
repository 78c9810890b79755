// ba_loop.h -- what bsfm_run_sfm_outlier_loop (ba_solver.cu) shares with the outlier pass (ba_outliers.cu) and the device
// compaction between rounds (ba_loop.cu).
#pragma once
#include "ba_setup.h"

namespace bsfm {
namespace ba {

struct CamCompact { double R[9], t[3], f, k0, k1; };
struct Rot3 { double R[9]; };

// Device camera tables of one outlier pass: what the loop of Bundle.cpp:721-754 reads of every camera
struct OutlierCams {
    CamCompact *cams = nullptr;
    CamIntrinsics *intr = nullptr;   // only when some camera is calibrated
    CamFisheye *fe = nullptr;        // only with optimize_for_fisheye
    Rot3 Rs = {};                    // GetRotationFromSpherical(-pi/2, pi/2), with fe
};
int upload_outlier_cams(const bsfm_camera_params_t *cams, int m, int optimize_for_fisheye, DeviceArena &D, OutlierCams &T);

// What one outlier pass leaves on the device
struct OutlierPass {
    double *dist = nullptr;     // nvis, in the order of the projections
    double *stats = nullptr;    // m x 5
    int *first_cam = nullptr;   // n: lowest camera that flags the point, or a value >= m
    double *err = nullptr;      // n: the distance in that camera (written for flagged points only)
};
// The pass itself on `st`: everything it reads is on the device already, nothing comes back to the host.
// d_prot (nullable, n): protected points.
int outliers_core(const Visibility &vis, int n, int m, const OutlierCams &T, const double *d_pts, const double *d_proj,
                  int estimate_distortion, double min_thresh, double max_thresh, const char *d_prot, cudaStream_t st, DeviceArena &D,
                  OutlierPass &out);

// The scene of one round of the outlier loop, on the device.  Point q of the round is point orig[q] of the call.
struct LoopScene {
    int n = 0, nvis = 0;
    int *vis_ptr = nullptr;     // n + 1
    int *vis_cam = nullptr;     // nvis
    double *proj = nullptr;     // 2 nvis
    double *p = nullptr;        // m cnp + 3 n: the solver's parameter vector (cameras, then points)
    int *orig = nullptr;        // n
    char *prot = nullptr;       // n, or null when no point is protected
};
// Capacity for n points and nvis observations
int alloc_loop_scene(LoopScene &S, int n, int nvis, int ncam_params, bool with_prot, DeviceArena &D);

// The arrays of the call, by original point index
struct LoopFull {
    double *pts = nullptr;        // num_pts x 3: every point as it was last solved (Bundle.cpp:905-909)
    int *pt_round = nullptr;      // num_pts
    double *pt_error = nullptr;   // num_pts
    const char *prot = nullptr;   // num_pts, or null
};

// Drops the points without views on entry (Bundle.cpp:614-636): src (the caller's CRS and projections, points read from
// full.pts) -> dst, and pt_round = -2 / -1, pt_error = 0.  counts (host, 3 ints) = { dst.n, dst.nvis, 0 }.  One
// synchronisation of st.
int loop_compact_entry(int num_pts, int ncam_params, const int *vis_ptr, const int *vis_cam, const double *proj, const LoopFull &full,
                       LoopScene &dst, int *counts, cudaStream_t st, DeviceArena &D);
// After a round's outlier pass: writes the round's points into full.pts by original index, and, with `remove`, records
// pt_round / pt_error of the flagged points and gathers the others into dst, renumbered densely in ascending order
// (Bundle.cpp:858-909).  counts (host, 3 ints) = { dst.n, dst.nvis, flagged points }.  One synchronisation of st.
int loop_compact_round(int m, int ncam_params, int round, int remove, const LoopScene &src, const OutlierPass &pass, const LoopFull &full,
                       LoopScene &dst, int *counts, cudaStream_t st, DeviceArena &D);

}  // namespace ba
}  // namespace bsfm
