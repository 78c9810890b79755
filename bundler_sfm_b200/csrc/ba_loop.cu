// ba_loop.cu -- the scene of bsfm_run_sfm_outlier_loop between two rounds, on the device (ba_loop.h): what
// BundlerApp::RunSFM_SBA does on the host around every run_sfm (src/Bundle.cpp:598-637, :858-909).
//   drop    : points without views leave the problem, the others are renumbered densely in ascending order (:614-636)
//   remove  : every view of a flagged point goes away (:871-889)
//   restore : init_pts[i] = nz_pts[remap[i]] for every point that was solved (:905-909)
// Every kernel is a gather or a scatter to distinct addresses, the two scans are integer sums and the one atomic counts
// integers: the result does not depend on the schedule.
#include <cub/device/device_scan.cuh>

#include "ba_loop.h"

namespace bsfm {
namespace ba {

// entry n of keep / cnt is the scans' total
__global__ void loop_entry_keep_kernel(int n, const int *vis_ptr, int *keep, int *cnt, int *pt_round, double *pt_error)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { keep[n] = 0; cnt[n] = 0; return; }
    const int views = vis_ptr[i + 1] - vis_ptr[i];
    keep[i] = views > 0;
    cnt[i] = views;
    pt_round[i] = views > 0 ? -1 : -2;
    pt_error[i] = 0.0;
}

// one thread per point q of the round: its refined position goes to the call's array by ORIGINAL index; a flagged point is
// counted and, when outliers are removed, recorded and left out of the next round
__global__ void loop_round_keep_kernel(int n, int m, int round, int remove, const int *vis_ptr, const int *first_cam, const double *err,
                                       const int *orig, const double *pts, double *full_pts, int *pt_round, double *pt_error,
                                       int *keep, int *cnt, int *flagged)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q > n) return;
    if (q == n) { keep[n] = 0; cnt[n] = 0; return; }
    const int o = orig[q];
    for (int c = 0; c < 3; c++) full_pts[3 * (size_t) o + c] = pts[3 * (size_t) q + c];
    const bool flag = first_cam[q] < m;
    if (flag) atomicAdd(flagged, 1);
    const bool gone = flag && remove;
    if (gone) { pt_round[o] = round; pt_error[o] = err[q]; }
    keep[q] = !gone;
    cnt[q] = gone ? 0 : vis_ptr[q + 1] - vis_ptr[q];
}

// one warp per point q: a kept point moves to new_idx[q] with its views at new_ptr[q]; warp n closes the row pointers and
// reports the new sizes.  orig == null: the source is the call's own numbering.
__global__ void loop_gather_kernel(int n, const int *vis_ptr, const int *vis_cam, const double *proj, const double *pts, const int *orig,
                                   const char *full_prot, const int *keep, const int *new_idx, const int *new_ptr,
                                   int *d_vis_ptr, int *d_vis_cam, double *d_proj, double *d_pts, int *d_orig, char *d_prot, int *counts)
{
    const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q > n) return;
    if (q == n) {
        if (lane == 0) { d_vis_ptr[new_idx[n]] = new_ptr[n]; counts[0] = new_idx[n]; counts[1] = new_ptr[n]; }
        return;
    }
    if (!keep[q]) return;
    const int nq = new_idx[q], s = vis_ptr[q], d = new_ptr[q], len = vis_ptr[q + 1] - s;
    if (lane == 0) {
        const int o = orig ? orig[q] : q;
        d_vis_ptr[nq] = d;
        d_orig[nq] = o;
        if (full_prot) d_prot[nq] = full_prot[o];
    }
    if (lane < 3) d_pts[3 * (size_t) nq + lane] = pts[3 * (size_t) q + lane];
    for (int v = lane; v < len; v += 32) {
        d_vis_cam[d + v] = vis_cam[s + v];
        d_proj[2 * (size_t) (d + v)] = proj[2 * (size_t) (s + v)];
        d_proj[2 * (size_t) (d + v) + 1] = proj[2 * (size_t) (s + v) + 1];
    }
}

int alloc_loop_scene(LoopScene &S, int n, int nvis, int ncam_params, bool with_prot, DeviceArena &D)
{
    TRY(D.alloc(&S.vis_ptr, (size_t) n + 1)); TRY(D.alloc(&S.vis_cam, (size_t) nvis)); TRY(D.alloc(&S.proj, (size_t) nvis * 2));
    TRY(D.alloc(&S.p, (size_t) ncam_params + (size_t) n * 3)); TRY(D.alloc(&S.orig, (size_t) n));
    if (with_prot) TRY(D.alloc(&S.prot, (size_t) n));
    return BSFM_OK;
}

namespace {
// scans of keep / cnt (n + 1 entries each), the gather into dst, and the sizes it reports
int scan_and_gather(int n, const int *vis_ptr, const int *vis_cam, const double *proj, const double *pts, const int *orig,
                    const char *full_prot, int *keep, int *cnt, int *d_counts, int ncam_params, LoopScene &dst, cudaStream_t st, DeviceArena &D)
{
    int *new_idx, *new_ptr;
    TRY(D.alloc(&new_idx, (size_t) n + 1)); TRY(D.alloc(&new_ptr, (size_t) n + 1));
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, keep, new_idx, n + 1, st); }));
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, cnt, new_ptr, n + 1, st); }));
    loop_gather_kernel<<<(unsigned) (((size_t) n + 1) * 32 + 255) / 256, 256, 0, st>>>(n, vis_ptr, vis_cam, proj, pts, orig, full_prot, keep, new_idx, new_ptr,
                                                                                    dst.vis_ptr, dst.vis_cam, dst.proj, dst.p + ncam_params, dst.orig,
                                                                                    dst.prot, d_counts);
    BSFM_KERNEL_CHECK();
    return BSFM_OK;
}
}  // namespace

int loop_compact_entry(int num_pts, int ncam_params, const int *vis_ptr, const int *vis_cam, const double *proj, const LoopFull &full,
                       LoopScene &dst, int *counts, cudaStream_t st, DeviceArena &D)
{
    int *keep, *cnt, *d_counts;
    TRY(D.alloc(&keep, (size_t) num_pts + 1)); TRY(D.alloc(&cnt, (size_t) num_pts + 1)); TRY(D.alloc(&d_counts, 3));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 3 * sizeof(int), st));
    loop_entry_keep_kernel<<<(num_pts + 1 + 255) / 256, 256, 0, st>>>(num_pts, vis_ptr, keep, cnt, full.pt_round, full.pt_error);
    BSFM_KERNEL_CHECK();
    TRY(scan_and_gather(num_pts, vis_ptr, vis_cam, proj, full.pts, nullptr, full.prot, keep, cnt, d_counts, ncam_params, dst, st, D));
    BSFM_CUDA_TRY(cudaMemcpyAsync(counts, d_counts, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    dst.n = counts[0]; dst.nvis = counts[1];
    return BSFM_OK;
}

int loop_compact_round(int m, int ncam_params, int round, int remove, const LoopScene &src, const OutlierPass &pass, const LoopFull &full,
                       LoopScene &dst, int *counts, cudaStream_t st, DeviceArena &D)
{
    const int n = src.n;
    int *keep, *cnt, *d_counts;
    TRY(D.alloc(&keep, (size_t) n + 1)); TRY(D.alloc(&cnt, (size_t) n + 1)); TRY(D.alloc(&d_counts, 3));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 3 * sizeof(int), st));
    loop_round_keep_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(n, m, round, remove, src.vis_ptr, pass.first_cam, pass.err, src.orig,
                                                                src.p + ncam_params, full.pts, full.pt_round, full.pt_error, keep, cnt,
                                                                d_counts + 2);
    BSFM_KERNEL_CHECK();
    if (remove)
        TRY(scan_and_gather(n, src.vis_ptr, src.vis_cam, src.proj, src.p + ncam_params, src.orig, full.prot, keep, cnt, d_counts, ncam_params,
                            dst, st, D));
    BSFM_CUDA_TRY(cudaMemcpyAsync(counts, d_counts, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    if (remove) { dst.n = counts[0]; dst.nvis = counts[1]; }
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm
