// ba_setup.h -- host side of the BA setup, shared by the LM solver (ba_solver.cu) and the outlier pass (ba_outliers.cu):
// pooled device memory, cub's two-phase calls, and the structures built once per call from the visibility.
#pragma once
#include <algorithm>
#include <utility>
#include <vector>
#include "common.h"
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"

#define TRY(expr) do { int rc__ = (expr); if (rc__ != BSFM_OK) return rc__; } while (0)

namespace bsfm {
namespace ba {

// Host-to-device traffic of the calling thread while `on` (bsfm_run_sfm_outlier_loop reports it per round): every copy of
// the BA setup whose source may be host memory goes through note_upload, which looks the pointer up and counts it when it
// is.  Off, it costs one branch.
struct UploadTally { bool on = false; long long bytes = 0, largest = 0; };
extern thread_local UploadTally t_uploads;
void count_upload(const void *src, size_t bytes);
inline void note_upload(const void *src, size_t bytes) { if (t_uploads.on) count_upload(src, bytes); }

// Device memory of one call, recycled through a process-wide pool of the current device's blocks.  The pool serves every
// thread, so the destructor waits for `st`, the stream that uses the blocks, before returning them: an error return with
// work in flight must not hand them to another call while that work still writes them.
struct DeviceArena {
    explicit DeviceArena(cudaStream_t s) : st(s) {}
    ~DeviceArena();
    DeviceArena(const DeviceArena &) = delete;
    DeviceArena &operator=(const DeviceArena &) = delete;
    template <typename T> int alloc(T **out, size_t count)
    {
        void *p;
        TRY(alloc_bytes(&p, std::max<size_t>(count, 1) * sizeof(T)));
        *out = (T *) p;
        return BSFM_OK;
    }
    // alloc + copy of `count` elements from host or device memory, on st
    template <typename T> int upload(T **out, const void *src, size_t count)
    {
        TRY(alloc(out, count));
        note_upload(src, count * sizeof(T));
        BSFM_CUDA_TRY(cudaMemcpyAsync((void *) *out, src, count * sizeof(T), cudaMemcpyDefault, st));
        return BSFM_OK;
    }
    // cub's two-phase call: call(temp, bytes) sizes its scratch (grown here, kept for later calls), then does the work
    // in `launches` kernels
    template <typename F> int cub(int launches, F call)
    {
        size_t need = 0;
        BSFM_CUDA_TRY(call(nullptr, need));
        if (need > scratch_bytes) { char *q; TRY(alloc(&q, need)); scratch = q; scratch_bytes = need; }
        BSFM_CUDA_TRY(call(scratch, need));
        count_launch(launches);
        return BSFM_OK;
    }
    const cudaStream_t st;

private:
    int alloc_bytes(void **out, size_t bytes);
    std::vector<std::pair<void *, size_t>> blocks;
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
};

// Which cameras see which points (idxij, sba_levmar.c:652-663); the arrays exist only when nvis > 0
struct Visibility {
    int nvis = 0;
    int *rowptr = nullptr;    // n + 1, point-major CRS
    int *obs_cam = nullptr;   // nvis, ascending camera within each point
    int *obs_pt = nullptr;    // nvis
    int *cam_obs = nullptr;   // nvis, observation ids grouped by camera, ascending point within each camera
    int *cam_ptr = nullptr;   // m + 1: camera j's observations are cam_obs[cam_ptr[j] .. cam_ptr[j + 1])
};
// Where a call's visibility comes from: the dense n x m mask of the reference interface, or the caller's own CRS arrays
// (the layout of Visibility::rowptr / obs_cam).  Host (pageable or pinned) or device pointers.  Inside the library also:
// device CRS arrays the library wrote itself (`ours`: used in place, not checked again), and, for the solver, a Visibility
// that has been built already (`built`).
struct VisSource {
    const char *vmask = nullptr;
    const int32_t *vis_ptr = nullptr;   // n + 1
    const int32_t *vis_cam = nullptr;   // nvis
    int nvis = 0;
    bool ours = false;
    const struct Visibility *built = nullptr;
    static VisSource mask(const char *vmask) { VisSource s; s.vmask = vmask; return s; }
    static VisSource crs(const int32_t *vis_ptr, const int32_t *vis_cam, int nvis)
    {
        VisSource s; s.vis_ptr = vis_ptr; s.vis_cam = vis_cam; s.nvis = nvis; return s;
    }
    static VisSource device_crs(const int32_t *vis_ptr, const int32_t *vis_cam, int nvis)
    {
        VisSource s = crs(vis_ptr, vis_cam, nvis); s.ours = true; return s;
    }
    static VisSource visibility(const Visibility *V) { VisSource s; s.built = V; return s; }
    bool present() const { return built || vmask || (vis_ptr && (vis_cam || nvis == 0)); }
};
// Visibility from either source.  Synchronises `st` at most once: to learn nvis of a mask scanned on the device, or to
// read the verdict on a caller's CRS.  A malformed CRS returns BSFM_ERR_ARG naming the lowest offending point
// (crs_check_kernel, ba_setup.cu); nothing but that check reads the caller's arrays before the verdict is known.
int build_visibility(const VisSource &src, int n, int m, cudaStream_t st, DeviceArena &D, Visibility &V);

// Schur structure of P's visibility: fills P.nblocks, blk_key, blk_start, tuples, nchunks, chunk_off and schur_part
int build_schur_structure(Problem &P, cudaStream_t st, DeviceArena &D);

// Camera order of the reduced camera system (ba_order.cu, bsfm_ba_camera_order): pos[j - mcon] = block position of free
// camera j; scores[0] / [1] = tiles the large Cholesky's trailing update keeps in the natural / RCM order.  Returns 1 when
// RCM is taken, 0 when the natural order is kept (then pos is the identity).
int camera_order(int m, int mcon, int cnp, const uint32_t *keys, int nblocks, std::vector<int> &pos, int64_t scores[2]);
// Applies it to P (sets P.cam_pos) when the system takes the large Cholesky path and RCM wins; BSFM_BA_CAMERA_ORDER=0 keeps
// the natural order.  Then plans the band factorisation of S in that order (chol_band_plan) and uploads the plan into `band`
// when it fits (otherwise band.env stays null and the panel path runs).  Reads P.blk_key back to the host (one
// synchronisation of st).
int apply_camera_order(Problem &P, int cnp, cudaStream_t st, DeviceArena &D, CholBand &band);
// a fitting band plan -> its device copy, in D
int upload_band_plan(const CholBandPlan &plan, DeviceArena &D, CholBand &band);

}  // namespace ba
}  // namespace bsfm
