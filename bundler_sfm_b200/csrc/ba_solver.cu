// ba_solver.cu -- host Levenberg-Marquardt controller + C ABI of the BA path.
//
// Mirrors, statement by statement where it decides anything:
//   sba_motstr_levmar_x     lib/sba-1.5/sba_levmar.c:457-2081  (controller quirks: SURVEY.md A.3)
//   run_sfm                 lib/sfm-driver/sfm.c:592-1003       (packing :652-703, unpacking :876-929)
// All array work runs in the sm_90a kernels of ba_kernels.cu / ba_chol.cu; the host only reads back
// one small scalar block per LM phase.  No CPU fallback.
#include "common.h"
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"
#include "../../include/bsfm_b200_ba.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

namespace bsfm {
namespace ba {
__global__ void cam_prep_kernel(Problem, const double *, int);
template <bool KI> __global__ void residual_kernel(Problem, const double *, double *, const double *, double);
template <bool KI> __global__ void jacobian_kernel(Problem, const double *, int);
__global__ void v_kernel(Problem, const double *, const double *);
__global__ void u_partial_kernel(Problem, const double *, int);
__global__ void u_final_kernel(Problem, const double *, int);
__global__ void grad_stats_kernel(Problem, const double *);
__global__ void penalty_kernel(Problem, const double *);
__global__ void vinv_kernel(Problem);
__global__ void schur_partial_kernel(Problem);
__global__ void schur_final_kernel(Problem);
__global__ void tuple_expand_kernel(const int2 *, const int *, int4 *, int);
__global__ void chunk_count_kernel(const int *, int, int *);
__global__ void zero_kernel(double *, size_t);
__global__ void backsub_kernel(Problem, const double *);
__global__ void update_kernel(Problem, const double *, double *);
__global__ void mot_solve_kernel(Problem);
__global__ void vmask_count_kernel(const char *, int, int, int *);
__global__ void vmask_fill_kernel(const char *, int, int, const int *, int *, int *);
__global__ void tuple_count_kernel(int, int, const int *, const int *, int *);
__global__ void tuple_fill_kernel(int, int, int, const int *, const int *, const int *, uint32_t *, int2 *);
__global__ void iota_kernel(int *, int);
__global__ void wout_scatter_kernel(Problem, double *);
__global__ void vinv_export_kernel(Problem);
int chol_solve(cudaStream_t, double *, double *, int, double *, double *, Scalars *);

__global__ void cam_ptr_kernel(const uint32_t *sorted_cam, int nvis, int m, int *cam_ptr)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > m) return;
    int lo = 0, hi = nvis;   // first position with cam >= j
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sorted_cam[mid] < (uint32_t) j) lo = mid + 1; else hi = mid;
    }
    cam_ptr[j] = lo;
}
// obs_pt from the CRS row pointers (the host-scanned visibility mask below): one warp per point
__global__ void csr_rows_kernel(const int *rowptr, int n, int *obs_pt)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    for (int q = rowptr[i] + lane; q < rowptr[i + 1]; q += 32) obs_pt[q] = i;
}

// host_scan_vmask (common.cpp): dense n x m visibility mask -> CRS on the host, see there

__global__ void cast_u32_kernel(const int *in, uint32_t *out, int count)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < count) out[q] = (uint32_t) in[q];
}
}  // namespace ba
}  // namespace bsfm

using namespace bsfm;
using namespace bsfm::ba;

#define SBA_ERROR_RC (-1)
static const double SBA_EPSILON_SQ = 1E-12 * 1E-12;      // sba_levmar.c:34-35
static const double SBA_ONE_THIRD = 0.3333333334;         // sba_levmar.c:37

namespace {

// Device blocks are recycled across solves (RunSFM_SBA calls run_sfm once per outlier round on a problem of
// nearly the same size, src/Bundle.cpp:586-913): cudaMalloc/cudaFree cost tens of microseconds each and a solve of the
// 50-camera configuration only takes milliseconds.  Blocks return to a per-process pool when a solve ends.
struct BlockPool {
    std::mutex mu;
    std::multimap<size_t, void *> free_blocks;   // capacity -> pointer
    size_t pooled_bytes = 0;
    int device = -1;
    void bind_device(int dev)   // blocks belong to one device: drop the pool when the caller switches GPUs
    {
        std::lock_guard<std::mutex> g(mu);
        if (dev == device) return;
        for (auto &kv : free_blocks) cudaFree(kv.second);
        free_blocks.clear(); pooled_bytes = 0; device = dev;
    }
    void *get(size_t bytes, size_t *cap_out)
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = free_blocks.lower_bound(bytes);
        if (it != free_blocks.end() && it->first <= bytes + bytes / 4 + 4096) {
            void *p = it->second; *cap_out = it->first; pooled_bytes -= it->first;
            free_blocks.erase(it);
            return p;
        }
        return nullptr;
    }
    void put(void *p, size_t cap)
    {
        std::lock_guard<std::mutex> g(mu);
        if (pooled_bytes + cap > ((size_t) 24 << 30)) { cudaFree(p); return; }   // bound what the pool may hold
        free_blocks.emplace(cap, p); pooled_bytes += cap;
    }
};
static BlockPool g_pool;

struct DeviceArena {
    std::vector<std::pair<void *, size_t>> blocks;
    ~DeviceArena() { for (auto &b : blocks) g_pool.put(b.first, b.second); }
    template <typename T> int alloc(T **out, size_t count)
    {
        size_t bytes = (std::max<size_t>(count, 1) * sizeof(T) + 255) & ~(size_t) 255;
        size_t cap = bytes;
        void *p = g_pool.get(bytes, &cap);
        if (!p) {
            cudaError_t e = cudaMalloc(&p, bytes);
            if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString(e)); return BSFM_ERR_CUDA; }
            cap = bytes;
        }
        blocks.push_back({p, cap});
        *out = (T *) p;
        return BSFM_OK;
    }
};

struct Timing {
    float ms[6] = {0, 0, 0, 0, 0, 0};
    int iterations = 0;
    int launches = 0;
};
thread_local Timing g_timing;

struct PhaseTimer {
    // accumulates device time per phase with event pairs; cheap (events only) and optional
    cudaStream_t st;
    bool on;
    std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;
    std::vector<cudaEvent_t> pool;
    PhaseTimer(cudaStream_t s, bool enable) : st(s), on(enable) {}
    ~PhaseTimer() { for (auto e : pool) cudaEventDestroy(e); }
    cudaEvent_t get() { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); return e; }
    void begin(int phase) { if (!on) return; cudaEvent_t a = get(), b = get(); cudaEventRecord(a, st); spans.push_back({phase, {a, b}}); }
    void end() { if (!on) return; cudaEventRecord(spans.back().second.second, st); }
    void collect(float *ms) {
        if (!on) return;
        for (auto &s : spans) { float t = 0; cudaEventElapsedTime(&t, s.second.first, s.second.second); ms[s.first] += t; }
    }
};

}  // namespace

// BSFM_BA_HOST_TIMING=1: wall-clock marks of the host path (stderr), to see where an end-to-end call spends its time
struct HostMarks {
    bool on = getenv("BSFM_BA_HOST_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
    void mark(const char *what)
    {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[ba host] %-28s +%8.3f ms  (%8.3f ms)\n", what, std::chrono::duration<double, std::milli>(now - last).count(),
                std::chrono::duration<double, std::milli>(now - t0).count());
        last = now;
    }
};

#define TRY(expr) do { int rc__ = (expr); if (rc__ != BSFM_OK) return rc__; } while (0)
// PDL launch of a BA kernel on stream `st`
#define BA_LAUNCH(kernel, grid, block, ...)                                                              \
    do {                                                                                                \
        BSFM_CUDA_TRY(launch_pdl(kernel, dim3(grid), dim3(block), st, __VA_ARGS__));                    \
        BSFM_KERNEL_CHECK();                                                                            \
    } while (0)

// Shared implementation of the two LM drivers.
//   mot == 0 : sba_motstr_levmar_x (cameras + points), p = (a_1..a_m, b_1..b_n)
//   mot == 1 : sba_mot_levmar_x (sba_levmar.c:2090-2690; cameras only), p = (a_1..a_m), the points are read from
//              `fixed_pts` (n x 3; what sfm_project_point3_mot takes from its adata, sfm.c:553-560) and never change
// init_params (nullable, m entries): the calibrated-camera fields (known_intrinsics, K_known, k_known) are read.
static int levmar_impl(int mot, const double *fixed_pts, int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                       const double *x, const double *covx, int mnp,
                       const bsfm_sfm_model_t *model, const bsfm_camera_params_t *init_params, int jac_mode,
                       int itmax, int verbose, const double opts[6], double info[10],
                       int use_constraints, const bsfm_camera_constraints_t *constraints,
                       int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                       double *Vout, double *Sout, double *Uout, double *Wout)
{
    clear_error();
    TRY(require_device());
    const char *const fname = mot ? "sba_mot_levmar_x" : "sba_motstr_levmar_x";
    if (n <= 0 || m <= 0 || mcon < 0 || mcon >= m || !vmask || !p || !x || !model || !opts || (mot && !fixed_pts)) {
        set_error("bsfm_sba_motstr_levmar_model: bad arguments (n=%d m=%d mcon=%d)", n, m, mcon);
        return BSFM_ERR_ARG;
    }
    if (pnp != 3 || mnp != 2 || cnp < 6 || cnp > 9 || cnp != 6 + (model->est_focal_length ? 1 : 0) + (model->undistort ? 2 : 0)) {
        set_error("bsfm_sba_motstr_levmar_model: unsupported block sizes cnp=%d pnp=%d mnp=%d for the sfm camera model", cnp, pnp, mnp);
        return BSFM_ERR_UNSUPPORTED;
    }
    if (covx) { set_error("bsfm_sba_motstr_levmar_model: covx != NULL is not supported (Bundler always passes NULL, sfm.c:821)"); return BSFM_ERR_UNSUPPORTED; }
    if ((Sout || Uout || Wout) && mcon != 0) { set_error("bsfm_sba_motstr_levmar_model: Sout/Uout/Wout export assumes mcon == 0 (as the reference does, sba_levmar.c:2017-2022)"); return BSFM_ERR_UNSUPPORTED; }
    if ((int64_t) m * m > 0xffffffffLL) { set_error("too many cameras"); return BSFM_ERR_ARG; }
    {
        const char *jm = getenv("BSFM_BA_JAC");
        if (jm && !strcmp(jm, "analytic")) jac_mode = BSFM_BA_JAC_ANALYTIC;
        if (jm && !strcmp(jm, "fd")) jac_mode = BSFM_BA_JAC_FD;
    }
    { int dev = 0; BSFM_CUDA_TRY(cudaGetDevice(&dev)); g_pool.bind_device(dev); }
    const long long launches0 = g_kernel_launches.load();
    // stream, events and the pinned scalar blocks are created once per thread and device and reused: driver
    // calls that allocate (cudaMallocHost, cudaStreamCreate, ...) serialise on a global lock and cost more than
    // an LM iteration of the 50-camera configuration
    struct SolverCtx { int device = -1; cudaStream_t st = nullptr; cudaEvent_t ev_begin = nullptr, ev_end = nullptr; Scalars *h_sc = nullptr; double *h_mu = nullptr; };
    static thread_local SolverCtx ctx;
    {
        int dev = 0;
        BSFM_CUDA_TRY(cudaGetDevice(&dev));
        if (ctx.device != dev) {
            if (ctx.st) { cudaStreamDestroy(ctx.st); cudaEventDestroy(ctx.ev_begin); cudaEventDestroy(ctx.ev_end); cudaFreeHost(ctx.h_sc); cudaFreeHost(ctx.h_mu); ctx = SolverCtx(); }
            BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&ctx.st, cudaStreamNonBlocking));
            BSFM_CUDA_TRY(cudaEventCreate(&ctx.ev_begin));
            BSFM_CUDA_TRY(cudaEventCreate(&ctx.ev_end));
            BSFM_CUDA_TRY(cudaMallocHost(&ctx.h_sc, sizeof(Scalars)));
            BSFM_CUDA_TRY(cudaMallocHost(&ctx.h_mu, sizeof(double)));
            ctx.device = dev;
        }
    }
    cudaStream_t st = ctx.st;
    const bool timing_on = getenv("BSFM_BA_TIMING") != nullptr;
    PhaseTimer PT(st, timing_on);
    cudaEvent_t ev_begin = ctx.ev_begin, ev_end = ctx.ev_end;
    BSFM_CUDA_TRY(cudaEventRecord(ev_begin, st));
    g_timing = Timing();
    HostMarks HM;

    DeviceArena D;
    Problem P;
    memset(&P, 0, sizeof P);
    P.n = n; P.m = m; P.mcon = mcon;
    P.M.cnp = cnp; P.M.est_focal = model->est_focal_length ? 1 : 0; P.M.undistort = model->undistort ? 1 : 0;
    P.M.explicit_centers = model->explicit_camera_centers ? 1 : 0;
    P.M.focal_idx = P.M.est_focal ? 6 : -1;
    P.M.k_idx = P.M.undistort ? (P.M.est_focal ? 7 : 6) : -1;
    P.M.f_scale = model->f_scale; P.M.k_scale = model->k_scale;
    P.nvars = m * cnp + n * 3;
    P.nlm = mot ? m * cnp : P.nvars;
    P.Sdim = (m - mcon) * cnp;

    // ---------------- setup: vmask -> CRS (sba_levmar.c:652-663), camera-major permutation ----------------
    PT.begin(0);
    char *d_vmask = nullptr; int *d_rowcnt, *d_rowptr;
    // host-resident masks of at least BSFM_BA_MASK_HOST_MIN bytes are scanned on the host and only their CRS form is uploaded
    // (host_scan_vmask above).  OFF by default: at config 3 it cuts the H2D bytes per solve from 560 to 75 MB, but the scan of the
    // 500 MB mask costs host time, and whether it beats the PCIe copy from pinned memory depends on the host.
    static const size_t host_scan_min = []() { const char *e = getenv("BSFM_BA_MASK_HOST_MIN"); return e ? (size_t) atoll(e) : ~(size_t) 0; }();
    bool host_mask = false;
    if ((size_t) n * m >= host_scan_min) {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, vmask) == cudaSuccess) host_mask = (pa.type == cudaMemoryTypeHost || pa.type == cudaMemoryTypeUnregistered);
        else cudaGetLastError();
    }
    std::vector<int> h_rowptr, h_obs_cam;
    TRY(D.alloc(&d_rowcnt, (size_t) n + 1));
    TRY(D.alloc(&d_rowptr, (size_t) n + 1));
    size_t cub_bytes = 0;
    void *d_cub = nullptr;
    auto ensure_cub = [&](size_t need) -> int {
        if (need <= cub_bytes) return BSFM_OK;
        char *q; int rc = D.alloc(&q, need); if (rc != BSFM_OK) return rc;
        d_cub = q; cub_bytes = need; return BSFM_OK;
    };
    if (host_mask) {
        bsfm::host_scan_vmask(vmask, n, m, h_rowptr, h_obs_cam);
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_rowptr, h_rowptr.data(), ((size_t) n + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    } else {
        TRY(D.alloc(&d_vmask, (size_t) n * m));
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_vmask, vmask, (size_t) n * m, cudaMemcpyDefault, st));   // host or device pointer (UVA)
        BSFM_CUDA_TRY(cudaMemsetAsync(d_rowcnt, 0, ((size_t) n + 1) * sizeof(int), st));
        vmask_count_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(d_vmask, n, m, d_rowcnt);
        BSFM_KERNEL_CHECK();
        size_t need = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, need, d_rowcnt, d_rowptr, n + 1, st);
        TRY(ensure_cub(need));
        cub::DeviceScan::ExclusiveSum(d_cub, need, d_rowcnt, d_rowptr, n + 1, st);
        count_launch(2);
    }
    int nvis = 0;
    if (host_mask) nvis = h_rowptr[n];
    else {
        BSFM_CUDA_TRY(cudaMemcpyAsync(&nvis, d_rowptr + n, sizeof(int), cudaMemcpyDeviceToHost, st));
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    }
    P.nvis = nvis;
    const int nobs = nvis * 2;
    if (nobs < P.nlm) {   // sba_levmar.c:647-650, :2235-2238
        fprintf(stderr, "SBA: %s() cannot solve a problem with fewer measurements [%d] than unknowns [%d]\n", fname, nobs, P.nlm);
        set_error("fewer measurements [%d] than unknowns [%d]", nobs, P.nlm);
        return SBA_ERROR_RC;
    }
    int *d_obs_cam, *d_obs_pt, *d_cam_ptr, *d_cam_obs, *d_iota;
    uint32_t *d_key_a, *d_key_b;
    TRY(D.alloc(&d_obs_cam, (size_t) nvis)); TRY(D.alloc(&d_obs_pt, (size_t) nvis));
    TRY(D.alloc(&d_cam_ptr, (size_t) m + 1)); TRY(D.alloc(&d_cam_obs, (size_t) nvis)); TRY(D.alloc(&d_iota, (size_t) nvis));
    if (host_mask) {
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_obs_cam, h_obs_cam.data(), (size_t) nvis * sizeof(int), cudaMemcpyHostToDevice, st));
        csr_rows_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(d_rowptr, n, d_obs_pt);
    } else {
        vmask_fill_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(d_vmask, n, m, d_rowptr, d_obs_cam, d_obs_pt);
    }
    BSFM_KERNEL_CHECK();
    double *d_x;
    TRY(D.alloc(&d_x, (size_t) nobs));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_x, x, (size_t) nobs * sizeof(double), cudaMemcpyDefault, st));
    // camera-major permutation: stable sort of observation ids by camera
    TRY(D.alloc(&d_key_a, (size_t) nvis)); TRY(D.alloc(&d_key_b, (size_t) nvis));
    cast_u32_kernel<<<(nvis + 255) / 256, 256, 0, st>>>(d_obs_cam, d_key_a, nvis);
    BSFM_KERNEL_CHECK();
    iota_kernel<<<(nvis + 255) / 256, 256, 0, st>>>(d_iota, nvis);
    BSFM_KERNEL_CHECK();
    {
        int bits = 1; while ((1LL << bits) < m) bits++;
        size_t need = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, need, d_key_a, d_key_b, d_iota, d_cam_obs, nvis, 0, bits, st);
        TRY(ensure_cub(need));
        cub::DeviceRadixSort::SortPairs(d_cub, need, d_key_a, d_key_b, d_iota, d_cam_obs, nvis, 0, bits, st);
        count_launch(3);
    }
    cam_ptr_kernel<<<(m + 1 + 255) / 256, 256, 0, st>>>(d_key_b, nvis, m, d_cam_ptr);
    BSFM_KERNEL_CHECK();

    // Schur structure: (obs_a, obs_b) tuples of every point, sorted by block key j*m+k (stable => ascending point)
    int *d_tcnt, *d_toff;
    TRY(D.alloc(&d_tcnt, (size_t) n + 1)); TRY(D.alloc(&d_toff, (size_t) n + 1));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_tcnt, 0, ((size_t) n + 1) * sizeof(int), st));
    tuple_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, mcon, d_rowptr, d_obs_cam, d_tcnt);
    BSFM_KERNEL_CHECK();
    {
        size_t need = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, need, d_tcnt, d_toff, n + 1, st);
        TRY(ensure_cub(need));
        cub::DeviceScan::ExclusiveSum(d_cub, need, d_tcnt, d_toff, n + 1, st);
        count_launch(2);
    }
    int ntuples = 0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(&ntuples, d_toff + n, sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    uint32_t *d_tkey_a, *d_tkey_b, *d_blk_key;
    unsigned long long *d_tval_a, *d_tval_b;
    int *d_blk_cnt, *d_blk_start, *d_nruns;
    TRY(D.alloc(&d_tkey_a, (size_t) ntuples)); TRY(D.alloc(&d_tkey_b, (size_t) ntuples));
    TRY(D.alloc(&d_tval_a, (size_t) ntuples)); TRY(D.alloc(&d_tval_b, (size_t) ntuples));
    const int max_blocks = (int) std::min<int64_t>((int64_t) ntuples, (int64_t) (m - mcon) * (m - mcon + 1) / 2);
    TRY(D.alloc(&d_blk_key, (size_t) max_blocks + 1)); TRY(D.alloc(&d_blk_cnt, (size_t) max_blocks + 1));
    TRY(D.alloc(&d_blk_start, (size_t) max_blocks + 2)); TRY(D.alloc(&d_nruns, 1));
    tuple_fill_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, m, mcon, d_rowptr, d_obs_cam, d_toff, d_tkey_a, (int2 *) d_tval_a);
    BSFM_KERNEL_CHECK();
    {
        int bits = 1; while ((1LL << bits) < (long long) m * m) bits++;
        size_t need = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, need, d_tkey_a, d_tkey_b, d_tval_a, d_tval_b, ntuples, 0, bits, st);
        TRY(ensure_cub(need));
        cub::DeviceRadixSort::SortPairs(d_cub, need, d_tkey_a, d_tkey_b, d_tval_a, d_tval_b, ntuples, 0, bits, st);
        count_launch(3);
        need = 0;
        cub::DeviceRunLengthEncode::Encode(nullptr, need, d_tkey_b, d_blk_key, d_blk_cnt, d_nruns, ntuples, st);
        TRY(ensure_cub(need));
        cub::DeviceRunLengthEncode::Encode(d_cub, need, d_tkey_b, d_blk_key, d_blk_cnt, d_nruns, ntuples, st);
        count_launch(2);
    }
    int nblocks = 0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(&nblocks, d_nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    {
        BSFM_CUDA_TRY(cudaMemsetAsync(d_blk_cnt + nblocks, 0, sizeof(int), st));
        size_t need = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, need, d_blk_cnt, d_blk_start, nblocks + 1, st);
        TRY(ensure_cub(need));
        cub::DeviceScan::ExclusiveSum(d_cub, need, d_blk_cnt, d_blk_start, nblocks + 1, st);
        count_launch(2);
    }
    P.rowptr = d_rowptr; P.obs_cam = d_obs_cam; P.obs_pt = d_obs_pt; P.cam_ptr = d_cam_ptr; P.cam_obs = d_cam_obs;
    // chunk list (SCHUR_CHUNK tuples per partial-sum warp) + (obs_a, obs_b, point) tuples
    int *d_chunk_cnt, *d_chunk_off;
    int4 *d_tuples4;
    TRY(D.alloc(&d_chunk_cnt, (size_t) nblocks + 1)); TRY(D.alloc(&d_chunk_off, (size_t) nblocks + 1));
    TRY(D.alloc(&d_tuples4, (size_t) ntuples));
    chunk_count_kernel<<<(nblocks + 1 + 255) / 256, 256, 0, st>>>(d_blk_cnt, nblocks, d_chunk_cnt);
    BSFM_KERNEL_CHECK();
    {
        size_t need = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, need, d_chunk_cnt, d_chunk_off, nblocks + 1, st);
        TRY(ensure_cub(need));
        cub::DeviceScan::ExclusiveSum(d_cub, need, d_chunk_cnt, d_chunk_off, nblocks + 1, st);
        count_launch(2);
    }
    tuple_expand_kernel<<<(ntuples + 255) / 256, 256, 0, st>>>((const int2 *) d_tval_b, d_obs_pt, d_tuples4, ntuples);
    BSFM_KERNEL_CHECK();
    int nchunks = 0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(&nchunks, d_chunk_off + nblocks, sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    P.nblocks = nblocks; P.blk_key = d_blk_key; P.blk_start = d_blk_start; P.tuples = d_tuples4;
    P.nchunks = nchunks; P.chunk_off = d_chunk_off;
    TRY(D.alloc(&P.schur_part, (size_t) nchunks * SCHUR_PART_STRIDE));
    P.x = d_x;

    // model + constraints
    double *d_Rinit, *d_ffixed;
    TRY(D.alloc(&d_Rinit, (size_t) m * 9)); TRY(D.alloc(&d_ffixed, (size_t) m));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_Rinit, model->R_init, (size_t) m * 9 * sizeof(double), cudaMemcpyHostToDevice, st));
    if (model->f_fixed) BSFM_CUDA_TRY(cudaMemcpyAsync(d_ffixed, model->f_fixed, (size_t) m * sizeof(double), cudaMemcpyHostToDevice, st));
    else BSFM_CUDA_TRY(cudaMemsetAsync(d_ffixed, 0, (size_t) m * sizeof(double), st));
    P.R_init = d_Rinit; P.f_fixed = d_ffixed;
    // calibrated cameras (sfm.c:339-357): the table exists only when one is present, and selects the KI kernels
    std::vector<CamIntrinsics> h_intr;
    if (init_params) {
        bool any_known = false;
        for (int j = 0; j < m && !any_known; j++) any_known = init_params[j].known_intrinsics != 0;
        if (any_known) {
            h_intr.resize(m);
            for (int j = 0; j < m; j++) h_intr[j] = cam_intrinsics(init_params[j]);
            CamIntrinsics *d_intr;
            TRY(D.alloc(&d_intr, (size_t) m));
            BSFM_CUDA_TRY(cudaMemcpyAsync(d_intr, h_intr.data(), (size_t) m * sizeof(CamIntrinsics), cudaMemcpyHostToDevice, st));
            P.intr = d_intr;
        }
    }
    auto *const k_residual = P.intr ? residual_kernel<true> : residual_kernel<false>;
    auto *const k_jacobian = P.intr ? jacobian_kernel<true> : jacobian_kernel<false>;
    std::vector<char> h_cc; std::vector<double> h_cv, h_cw;
    if (use_constraints) {
        if (!constraints) { set_error("use_constraints set but constraints == NULL"); return BSFM_ERR_ARG; }
        h_cc.resize((size_t) m * cnp); h_cv.resize((size_t) m * cnp); h_cw.resize((size_t) m * cnp);
        for (int j = 0; j < m; j++)
            for (int q = 0; q < cnp; q++) {
                h_cc[(size_t) j * cnp + q] = constraints[j].constrained[q] ? 1 : 0;
                h_cv[(size_t) j * cnp + q] = constraints[j].constraints[q];
                h_cw[(size_t) j * cnp + q] = constraints[j].weights[q];
            }
        char *dc; double *dv, *dw;
        TRY(D.alloc(&dc, h_cc.size())); TRY(D.alloc(&dv, h_cv.size())); TRY(D.alloc(&dw, h_cw.size()));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dc, h_cc.data(), h_cc.size(), cudaMemcpyHostToDevice, st));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dv, h_cv.data(), h_cv.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dw, h_cw.data(), h_cw.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        P.cam_constrained = dc; P.cam_constraints = dv; P.cam_weights = dw;
    }
    std::vector<char> h_pc; std::vector<double> h_pv, h_pw;
    if (use_point_constraints) {
        if (!point_constraints) { set_error("use_point_constraints set but point_constraints == NULL"); return BSFM_ERR_ARG; }
        h_pc.resize(n); h_pv.resize((size_t) n * 3); h_pw.resize(n);
        for (int i = 0; i < n; i++) {
            h_pc[i] = point_constraints[i].constrained ? 1 : 0;
            for (int q = 0; q < 3; q++) h_pv[(size_t) i * 3 + q] = point_constraints[i].constraints[q];
            h_pw[i] = point_constraints[i].weight;
        }
        char *dc; double *dv, *dw;
        TRY(D.alloc(&dc, h_pc.size())); TRY(D.alloc(&dv, h_pv.size())); TRY(D.alloc(&dw, h_pw.size()));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dc, h_pc.data(), h_pc.size(), cudaMemcpyHostToDevice, st));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dv, h_pv.data(), h_pv.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        BSFM_CUDA_TRY(cudaMemcpyAsync(dw, h_pw.data(), h_pw.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        P.pt_constrained = dc; P.pt_constraints = dv; P.pt_weights = dw;
    }

    // work arrays
    const int Sdim = P.Sdim;
    double *d_p, *d_pdp, *d_e, *d_enew, *d_camR_a, *d_camR_b, *d_linv, *d_da;
    TRY(D.alloc(&d_p, (size_t) P.nvars)); TRY(D.alloc(&d_pdp, (size_t) P.nvars));
    TRY(D.alloc(&d_e, (size_t) nobs)); TRY(D.alloc(&d_enew, (size_t) nobs));
    TRY(D.alloc(&d_camR_a, (size_t) m * 36)); TRY(D.alloc(&d_camR_b, (size_t) m * 36));
    TRY(D.alloc(&P.jacA, (size_t) nvis * 2 * cnp)); TRY(D.alloc(&P.jacB, (size_t) nvis * 6));
    TRY(D.alloc(&P.W, (size_t) nvis * cnp * 3));
    TRY(D.alloc(&P.U, (size_t) m * cnp * cnp)); TRY(D.alloc(&P.V, (size_t) n * 9)); TRY(D.alloc(&P.Vinv, (size_t) n * 9));
    TRY(D.alloc(&P.eab, (size_t) P.nvars)); TRY(D.alloc(&P.dp, (size_t) P.nvars));
    TRY(D.alloc(&P.S, ((size_t) Sdim + 1) * Sdim));
    P.E = P.S + (size_t) Sdim * Sdim;      // RHS lives in matrix row Sdim (see ba_chol.cu)
    double *d_Lmat;
    TRY(D.alloc(&d_Lmat, ((size_t) Sdim + 1) * Sdim));   // Cholesky factor (out of place)
    TRY(D.alloc(&d_linv, (size_t) ((Sdim + 31) / 32) * 1024 + chol_extra_ws_doubles(Sdim))); TRY(D.alloc(&d_da, (size_t) Sdim));
    const int red_blocks_obs = (nvis + 255) / 256, red_blocks_var = (P.nvars + 255) / 256;
    TRY(D.alloc(&P.partial, (size_t) 3 * std::max(red_blocks_obs, red_blocks_var) + 8));
    const int useg = std::max(1, std::min(32, (nvis / m + 1023) / 1024));   // ~1024 observations per U-accumulation CTA
    TRY(D.alloc(&P.u_part, (size_t) m * useg * 54));
    TRY(D.alloc(&P.ticket, 4));
    BSFM_CUDA_TRY(cudaMemsetAsync(P.ticket, 0, 4 * sizeof(unsigned int), st));
    TRY(D.alloc(&P.sc, 1));
    BSFM_CUDA_TRY(cudaMemsetAsync(P.sc, 0, sizeof(Scalars), st));
    double *d_mu, *h_mu = ctx.h_mu;
    TRY(D.alloc(&d_mu, 1));
    P.mu = d_mu;
    Scalars *h_sc = ctx.h_sc;
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_p, p, (size_t) P.nlm * sizeof(double), cudaMemcpyDefault, st));
    if (mot) {
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_p + P.nlm, fixed_pts, (size_t) n * 3 * sizeof(double), cudaMemcpyDefault, st));
        BSFM_CUDA_TRY(cudaMemsetAsync(P.dp, 0, (size_t) P.nvars * sizeof(double), st));   // the points' increments stay 0
    }
    PT.end();
    HM.mark("setup issued");

    auto read_scalars = [&]() -> int {
        BSFM_CUDA_TRY(cudaMemcpyAsync(h_sc, P.sc, sizeof(Scalars), cudaMemcpyDeviceToHost, st));
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));
        return BSFM_OK;
    };
    const int with_pert = (jac_mode == BSFM_BA_JAC_FD) ? 1 : 0;
    auto launch_residual = [&](const double *pp, double *camR, double *eout, const double *eprev, double eps5v) -> int {
        P.camR = camR;
        BA_LAUNCH(cam_prep_kernel, (m + 127) / 128, 128, P, pp, with_pert);
        BA_LAUNCH(k_residual, red_blocks_obs, 256, P, pp, eout, eprev, eps5v);
        return BSFM_OK;
    };

    // ---------------- LM controller (sba_levmar.c:603-2052) ----------------
    const double tau = fabs(opts[0]), eps1 = fabs(opts[1]), eps2 = fabs(opts[2]), eps2_sq = opts[2] * opts[2],
                 eps3_sq = opts[3] * opts[3], eps4_sq = opts[4] * opts[4], eps5 = opts[5];
    double mu = 0.0, eab_inf = 0.0, p_eL2, pdp_eL2, p_L2 = 0.0, dp_L2 = DBL_MAX, dF, dL, init_p_eL2, max_diag = DBL_MIN, pen = 0.0;
    int nu = 2, nu2, stop = 0, nfev = 0, njev = 0, nlss = 0, itno = 0;
    const bool any_constraints = use_constraints || use_point_constraints;
    bool almost_singular = false;
    const bool s_dense = (int64_t) nblocks == (int64_t) (m - mcon) * (m - mcon + 1) / 2;   // every block written by the Schur pass

    PT.begin(4);
    TRY(launch_residual(d_p, d_camR_a, d_e, nullptr, 0.0)); nfev = 1;
    if (any_constraints) { BA_LAUNCH(penalty_kernel, 1, 32, P, d_p); BSFM_KERNEL_CHECK(); }
    PT.end();
    TRY(read_scalars());
    pen = any_constraints ? h_sc->penalty : 0.0;
    p_eL2 = h_sc->e_L2 + pen;    // sba_levmar.c:802-842
    if (verbose) printf(mot ? "initial mot-SBA error %g [%g]\n" : "initial motstr-SBA error %g [%g]\n", p_eL2, p_eL2 / nvis);
    init_p_eL2 = p_eL2;
    if (!std::isfinite(p_eL2)) stop = 7;

    HM.mark("initial residual");
    for (itno = 0; itno < itmax && !stop; ++itno) {
        PT.begin(1);
        P.camR = d_camR_a;
        k_jacobian<<<(nvis + 127) / 128, 128, 0, st>>>(P, d_p, jac_mode); ++njev;
        BSFM_KERNEL_CHECK();
        u_partial_kernel<<<m * useg, 128, 0, st>>>(P, d_e, useg);
        BA_LAUNCH(u_final_kernel, m, 96, P, d_p, useg);
        if (!mot) BA_LAUNCH(v_kernel, (n + 127) / 128, 128, P, d_p, d_e);
        if (Vout) BSFM_CUDA_TRY(cudaMemcpyAsync(Vout, P.V, (size_t) n * 9 * sizeof(double), cudaMemcpyDefault, st));   // :1039-1051
        BA_LAUNCH(grad_stats_kernel, red_blocks_var, 256, P, d_p);
        PT.end();
        TRY(read_scalars());
        eab_inf = h_sc->eab_inf; p_L2 = h_sc->p_L2; max_diag = h_sc->max_diag;
        if (any_constraints) pen = h_sc->penalty;

        if (eab_inf <= eps1) { dp_L2 = 0.0; stop = 1; break; }      // :1117-1121
        if (itno == 0) mu = tau * max_diag;                          // :1123-1128

        while (1) {   // damping loop :1131
            BSFM_CUDA_TRY(cudaMemsetAsync(&P.sc->singular_v, 0, 3 * sizeof(int), st));
            *h_mu = mu;
            BSFM_CUDA_TRY(cudaMemcpyAsync(d_mu, h_mu, sizeof(double), cudaMemcpyHostToDevice, st));
            if (mot) {
                // block-diagonal system: (U_j + mu I) da_j = ea_j per camera (sba_levmar.c:2487-2514)
                PT.begin(3);
                BA_LAUNCH(mot_solve_kernel, (m + 63) / 64, 64, P);
                PT.end();
                PT.begin(4);
            } else {
            PT.begin(2);
            BA_LAUNCH(vinv_kernel, (n + 255) / 256, 256, P);
            if (!s_dense) {   // camera pairs without a common point keep S_jk = 0
                BA_LAUNCH(zero_kernel, std::min(1024, (int) (((size_t) Sdim * Sdim + 255) / 256)), 256, P.S, (size_t) Sdim * Sdim);
            }
            BA_LAUNCH(schur_partial_kernel, (nchunks * 32 + 127) / 128, 128, P);
            BA_LAUNCH(schur_final_kernel, (nblocks * 32 + 127) / 128, 128, P);
            PT.end();
            PT.begin(3);
            TRY(chol_solve(st, P.S, d_Lmat, Sdim, d_linv, d_da, P.sc));
            PT.end();
            PT.begin(4);
            BA_LAUNCH(backsub_kernel, (std::max(n, m * cnp) + 127) / 128, 128, P, d_da);
            }
            BA_LAUNCH(update_kernel, red_blocks_var, 256, P, d_p, d_pdp);
            TRY(launch_residual(d_pdp, d_camR_b, d_enew, d_e, eps5));
            PT.end();
            TRY(read_scalars());

            bool take_moredamping = true;
            if (!mot && h_sc->singular_v) {
                fprintf(stderr, "SBA: singular matrix V*_i in sba_motstr_levmar_x(), increasing damping\n");   // :1156-1161
            } else {
                nlss += mot ? (m - mcon) : 1;      // the motion-only routine counts one system per camera (:2513)
                const bool issolved = !h_sc->chol_fail;
                if (issolved) {
                    dp_L2 = h_sc->dp_L2;
                    if (dp_L2 <= eps2_sq * p_L2) { stop = 2; break; }                              // :1450-1454
                    if (dp_L2 >= (p_L2 + eps2) / SBA_EPSILON_SQ) {                                 // :1456-1462
                        fprintf(stderr, "SBA: the matrix of the augmented normal equations is almost singular in %s(),\n"
                                        "     minimization should be restarted from the current solution with an increased damping term\n", fname);
                        set_error("augmented normal equations almost singular");
                        // the reference leaves through freemem_and_return with the last ACCEPTED p in place (it updates p
                        // in place on every accepted step, sba_levmar.c:1456-1462): fall through to the common tail
                        almost_singular = true;
                        break;
                    }
                    ++nfev;
                    pdp_eL2 = h_sc->e_L2;
                    if (verbose > 1) printf("mean reprojection error (trial) sq %g\n", pdp_eL2 / nvis);
                    if (!std::isfinite(pdp_eL2)) { stop = 7; break; }                              // :1479-1485
                    pdp_eL2 += pen;   // constraint terms evaluated at the OLD p (quirk 7, :1487-1522)
                    dL = h_sc->dL;
                    dF = p_eL2 - pdp_eL2;
                    if (verbose > 1) {
                        printf("\ndamping term %8g, gain ratio %8g, errors %8g / %8g = %g\n", mu, dL != 0.0 ? dF / dL : dF / DBL_EPSILON,
                               p_eL2 / nvis, pdp_eL2 / nvis, p_eL2 / pdp_eL2);
                        printf("pdp_eL2: %0.3f, nvis: %d\n", pdp_eL2, nvis);
                    }
                    if (dL > 0.0 && dF > 0.0) {                                                    // :1543
                        double tmp = (2.0 * dF / dL - 1.0);
                        tmp = 1.0 - tmp * tmp * tmp;
                        mu = mu * ((tmp >= SBA_ONE_THIRD) ? tmp : SBA_ONE_THIRD);
                        nu = 2;
                        const double max_pct_change = h_sc->max_pct;
                        if (!mot) {     // Snavely's stop-8 statistic exists only in the motion+structure routine
                            printf("max_pct_change: %0.3e\n", max_pct_change);                     // :1563 (unconditional)
                            fflush(stdout);
                        }
                        if (pdp_eL2 - 2.0 * sqrt(p_eL2 * pdp_eL2) < (eps4_sq - 1.0) * p_eL2) stop = 4;   // :1567, :2596
                        if (!mot && max_pct_change < eps5 && itno >= 4) { stop = 8; break; }       // :1569-1572 (step discarded)
                        std::swap(d_p, d_pdp); std::swap(d_e, d_enew); std::swap(d_camR_a, d_camR_b);
                        p_eL2 = pdp_eL2;
                        if (any_constraints) { BA_LAUNCH(penalty_kernel, 1, 32, P, d_p); BSFM_KERNEL_CHECK(); }
                        take_moredamping = false;
                    }
                }
            }
            if (!take_moredamping) break;
            if (almost_singular) break;
            // moredamping :1584-1597
            mu *= nu;
            nu2 = nu << 1;
            if (nu2 <= nu) {
                fprintf(stderr, "SBA: too many failed attempts to increase the damping factor in %s()! Singular Hessian matrix?\n", fname);
                stop = 6;
                break;
            }
            nu = nu2;
        }
        if (almost_singular) break;
        if (p_eL2 <= eps3_sq) stop = 5;    // :1614
    }
    if (itno >= itmax) stop = 3;
    HM.mark("LM loop");

    if (Sout) {
        // export pass (sba_levmar.c:1633-2026): Jacobian at the final p, U/V/W with constraints, UNDAMPED Schur complement
        P.camR = d_camR_a;
        k_jacobian<<<(nvis + 127) / 128, 128, 0, st>>>(P, d_p, jac_mode); ++njev;
        BSFM_KERNEL_CHECK();
        u_partial_kernel<<<m * useg, 128, 0, st>>>(P, d_e, useg);
        BA_LAUNCH(u_final_kernel, m, 96, P, d_p, useg);
        BA_LAUNCH(v_kernel, (n + 127) / 128, 128, P, d_p, d_e);
        if (Uout) BSFM_CUDA_TRY(cudaMemcpyAsync(Uout, P.U, (size_t) m * cnp * cnp * sizeof(double), cudaMemcpyDefault, st));
        if (Vout) BSFM_CUDA_TRY(cudaMemcpyAsync(Vout, P.V, (size_t) n * 9 * sizeof(double), cudaMemcpyDefault, st));
        vinv_export_kernel<<<(n + 255) / 256, 256, 0, st>>>(P);
        BSFM_KERNEL_CHECK();
        if (Wout) {
            double *d_wout;
            TRY(D.alloc(&d_wout, (size_t) m * cnp * 3 * (size_t) n));
            BSFM_CUDA_TRY(cudaMemcpyAsync(d_wout, Wout, (size_t) m * cnp * 3 * (size_t) n * sizeof(double), cudaMemcpyDefault, st));   // untouched entries keep the caller's values
            wout_scatter_kernel<<<(nvis + 255) / 256, 256, 0, st>>>(P, d_wout);
            BSFM_KERNEL_CHECK();
            BSFM_CUDA_TRY(cudaMemcpyAsync(Wout, d_wout, (size_t) m * cnp * 3 * (size_t) n * sizeof(double), cudaMemcpyDefault, st));
        }
        *h_mu = 0.0;
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_mu, h_mu, sizeof(double), cudaMemcpyHostToDevice, st));
        BA_LAUNCH(zero_kernel, std::min(1024, (int) (((size_t) Sdim * Sdim + 255) / 256)), 256, P.S, (size_t) Sdim * Sdim);
        BA_LAUNCH(schur_partial_kernel, (nchunks * 32 + 127) / 128, 128, P);
        BA_LAUNCH(schur_final_kernel, (nblocks * 32 + 127) / 128, 128, P);
        BSFM_CUDA_TRY(cudaMemcpyAsync(Sout, P.S, (size_t) Sdim * Sdim * sizeof(double), cudaMemcpyDefault, st));   // symmetric: transpose == itself (:2017-2025)
    }
    BSFM_CUDA_TRY(cudaMemcpyAsync(p, d_p, (size_t) P.nlm * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaEventRecord(ev_end, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    if (info) {   // :2028-2049
        info[0] = init_p_eL2; info[1] = p_eL2; info[2] = eab_inf; info[3] = dp_L2;
        info[4] = mu / max_diag; info[5] = itno; info[6] = stop; info[7] = nfev; info[8] = njev; info[9] = nlss;
    }
    cudaEventElapsedTime(&g_timing.ms[5], ev_begin, ev_end);
    PT.collect(g_timing.ms);
    g_timing.iterations = itno;
    g_timing.launches = (int) (g_kernel_launches.load() - launches0);
    HM.mark("copy back + teardown");
    return (stop != 7 && !almost_singular) ? itno : SBA_ERROR_RC;
}

extern "C" int bsfm_sba_motstr_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                               const double *x, const double *covx, int mnp,
                                               const bsfm_sfm_model_t *model, int jac_mode,
                                               int itmax, int verbose, const double opts[6], double info[10],
                                               int use_constraints, const bsfm_camera_constraints_t *constraints,
                                               int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                               double *Vout, double *Sout, double *Uout, double *Wout,
                                               const bsfm_camera_params_t *init_params)
{
    return levmar_impl(0, nullptr, n, m, mcon, vmask, p, cnp, pnp, x, covx, mnp, model, init_params, jac_mode, itmax, verbose, opts, info,
                       use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout);
}

extern "C" int bsfm_sba_motstr_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                            const double *x, const double *covx, int mnp,
                                            const bsfm_sfm_model_t *model, int jac_mode,
                                            int itmax, int verbose, const double opts[6], double info[10],
                                            int use_constraints, const bsfm_camera_constraints_t *constraints,
                                            int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                            double *Vout, double *Sout, double *Uout, double *Wout)
{
    return bsfm_sba_motstr_levmar_model_ki(n, m, mcon, vmask, p, cnp, pnp, x, covx, mnp, model, jac_mode, itmax, verbose, opts, info,
                                           use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout,
                                           nullptr);
}

extern "C" int bsfm_sba_mot_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                            const double *x, const double *covx, int mnp,
                                            const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                            int itmax, int verbose, const double opts[6], double info[10],
                                            int use_constraints, const bsfm_camera_constraints_t *constraints,
                                            const bsfm_camera_params_t *init_params)
{
    return levmar_impl(1, points, n, m, mcon, vmask, p, cnp, 3, x, covx, mnp, model, init_params, jac_mode, itmax, verbose, opts, info,
                       use_constraints, constraints, 0, nullptr, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int bsfm_sba_mot_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                         const double *x, const double *covx, int mnp,
                                         const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                         int itmax, int verbose, const double opts[6], double info[10],
                                         int use_constraints, const bsfm_camera_constraints_t *constraints)
{
    return bsfm_sba_mot_levmar_model_ki(n, m, mcon, vmask, p, cnp, x, covx, mnp, model, points, jac_mode, itmax, verbose, opts, info,
                                        use_constraints, constraints, nullptr);
}

// == sba_Axb_Chol, lib/sba-1.5/sba_lapack.c:374-485: x = A^-1 B for symmetric positive definite A (m x m).
// A, B, x may be host or device pointers; A and B are never modified (the reference overwrites them when
// iscolmaj == 1; a symmetric matrix reads the same in both orders, so the flag changes nothing else here).
// Returns 1 on success, 0 when a leading minor is not positive definite (the reference's return values), < 0 on a
// library error.  `reps` > 1 repeats the factorisation on a fresh copy of A; *ms_out = device time per repetition.
static int axb_chol_impl(const double *A, const double *B, double *x, int m, int reps, float *ms_out)
{
    clear_error();
    TRY(require_device());
    if (!A || !B || !x || m <= 0 || reps < 1) { set_error("bsfm_sba_Axb_Chol: bad arguments"); return BSFM_ERR_ARG; }
    { int dev = 0; BSFM_CUDA_TRY(cudaGetDevice(&dev)); g_pool.bind_device(dev); }
    DeviceArena D;
    cudaStream_t st;
    BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamDestroy(s); } } guard{st};
    double *d_src, *d_A, *d_L, *d_linv, *d_x; Scalars *d_sc;
    const size_t mm = (size_t) m * m;
    TRY(D.alloc(&d_src, mm + m)); TRY(D.alloc(&d_A, mm + m)); TRY(D.alloc(&d_L, mm + m));
    TRY(D.alloc(&d_linv, (size_t) ((m + 31) / 32) * 1024 + chol_extra_ws_doubles(m))); TRY(D.alloc(&d_x, (size_t) m)); TRY(D.alloc(&d_sc, 1));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_src, A, mm * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_src + mm, B, (size_t) m * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_sc, 0, sizeof(Scalars), st));
    cudaEvent_t e0, e1;
    BSFM_CUDA_TRY(cudaEventCreate(&e0)); BSFM_CUDA_TRY(cudaEventCreate(&e1));
    float total = 0.f;
    int rc = BSFM_OK;
    for (int r = 0; r < reps && rc == BSFM_OK; r++) {
        cudaMemcpyAsync(d_A, d_src, (mm + m) * sizeof(double), cudaMemcpyDeviceToDevice, st);
        cudaEventRecord(e0, st);
        rc = chol_solve(st, d_A, d_L, m, d_linv, d_x, d_sc);
        cudaEventRecord(e1, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { set_error("bsfm_sba_Axb_Chol: %s", cudaGetErrorString(cudaGetLastError())); rc = BSFM_ERR_CUDA; }
        float t = 0.f; cudaEventElapsedTime(&t, e0, e1); total += t;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (rc != BSFM_OK) return rc;
    if (ms_out) *ms_out = total / reps;
    Scalars h;
    BSFM_CUDA_TRY(cudaMemcpy(&h, d_sc, sizeof h, cudaMemcpyDeviceToHost));
    if (h.chol_fail) return 0;
    BSFM_CUDA_TRY(cudaMemcpy(x, d_x, (size_t) m * sizeof(double), cudaMemcpyDefault));
    return 1;
}
extern "C" int bsfm_sba_Axb_Chol(const double *A, const double *B, double *x, int m, int iscolmaj)
{
    (void) iscolmaj;
    return axb_chol_impl(A, B, x, m, 1, nullptr);
}
extern "C" int bsfm_sba_Axb_Chol_timed(const double *A, const double *B, double *x, int m, int reps, float *ms_per_solve)
{
    return axb_chol_impl(A, B, x, m, reps, ms_per_solve);
}

extern "C" int bsfm_ba_last_timing(float ms[6], int *iterations, int *launches)
{
    if (ms) for (int q = 0; q < 6; q++) ms[q] = g_timing.ms[q];
    if (iterations) *iterations = g_timing.iterations;
    if (launches) *launches = g_timing.launches;
    return BSFM_OK;
}

// == run_sfm, lib/sfm-driver/sfm.c:592-1003
extern "C" int bsfm_run_sfm(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
                            int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                            bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                            int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                            double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                            double *Vout, double *Sout, double *Uout, double *Wout, double *info_out)
{
    clear_error();
    if (fix_points && (Vout || Sout || Uout || Wout)) { set_error("bsfm_run_sfm: fix_points=1 has no V/S/U/W export (nor has the reference, sfm.c:843-856)"); return BSFM_ERR_UNSUPPORTED; }
    if (optimize_for_fisheye) { set_error("bsfm_run_sfm: optimize_for_fisheye=1 is outside the GPU path"); return BSFM_ERR_UNSUPPORTED; }
    if (est_focal_length && const_focal_length) { set_error("bsfm_run_sfm: const_focal_length is not implemented (nor in the reference, sfm.c:518-521)"); return BSFM_ERR_UNSUPPORTED; }
    if (num_pts <= 0 || num_cameras <= 0 || !vmask || !projections || !init_camera_params || !init_pts) {
        set_error("bsfm_run_sfm: bad arguments"); return BSFM_ERR_ARG;
    }

    const double f_scale = 0.001, k_scale = 5.0;                 // sfm.c:634-635 (TEST_FOCAL)
    int cnp = est_focal_length ? 7 : 6;
    if (undistort) cnp += 2;
    const int num_camera_params = cnp * num_cameras;
    const size_t num_params = (size_t) num_camera_params + 3 * (size_t) num_pts;
    std::vector<double> params(num_params);
    std::vector<double> R_init((size_t) num_cameras * 9), f_fixed(num_cameras);
    for (int j = 0; j < num_cameras; j++) {                      // sfm.c:652-696
        int c;
        init_camera_params[j].f_scale = f_scale;
        init_camera_params[j].k_scale = k_scale;
        params[(size_t) cnp * j + 0] = init_camera_params[j].t[0];
        params[(size_t) cnp * j + 1] = init_camera_params[j].t[1];
        params[(size_t) cnp * j + 2] = init_camera_params[j].t[2];
        params[(size_t) cnp * j + 3] = 0.0; params[(size_t) cnp * j + 4] = 0.0; params[(size_t) cnp * j + 5] = 0.0;
        if (est_focal_length) { params[(size_t) cnp * j + 6] = init_camera_params[j].f * init_camera_params[j].f_scale; c = 7; }
        else c = 6;
        if (undistort) {
            const double scale = init_camera_params[j].k_scale;
            params[(size_t) cnp * j + c] = init_camera_params[j].k[0] * scale;
            params[(size_t) cnp * j + c + 1] = init_camera_params[j].k[1] * scale;
        }
        memcpy(&R_init[(size_t) j * 9], init_camera_params[j].R, 9 * sizeof(double));
        f_fixed[j] = init_camera_params[j].f;
    }
    for (int i = 0; i < num_pts; i++)                            // sfm.c:698-703
        for (int q = 0; q < 3; q++) params[(size_t) num_camera_params + 3 * (size_t) i + q] = init_pts[i].p[q];

    double opts[6] = {1.0e-3, 1.0e-10, eps2, 1.0e-12, 0.0, 4.0e-2};   // sfm.c:705-714
    double info[10] = {0};

    std::vector<bsfm_camera_constraints_t> constraints;
    std::vector<char> cc; std::vector<double> cv, cw;
    if (use_constraints) {                                       // sfm.c:721-754
        constraints.resize(num_cameras);
        cc.resize((size_t) num_cameras * cnp); cv.resize((size_t) num_cameras * cnp); cw.resize((size_t) num_cameras * cnp);
        for (int i = 0; i < num_cameras; i++) {
            char *c0 = &cc[(size_t) i * cnp]; double *v0 = &cv[(size_t) i * cnp]; double *w0 = &cw[(size_t) i * cnp];
            memcpy(c0, init_camera_params[i].constrained, cnp);
            memcpy(v0, init_camera_params[i].constraints, cnp * sizeof(double));
            memcpy(w0, init_camera_params[i].weights, cnp * sizeof(double));
            if (est_focal_length) { v0[6] *= f_scale; w0[6] *= (1.0 / (f_scale * f_scale)); }
            if (undistort) {
                // NOTE the reference indexes 7 and 8 unconditionally (sfm.c:745-751), i.e. it assumes est_focal_length;
                // with est_focal_length == 0 that would be out of bounds for cnp == 8, so the k pair at 6,7 is used there.
                const int k0 = est_focal_length ? 7 : 6;
                v0[k0] *= k_scale; w0[k0] *= (1.0 / (k_scale * k_scale));
                v0[k0 + 1] *= k_scale; w0[k0 + 1] *= (1.0 / (k_scale * k_scale));
            }
            constraints[i].constrained = c0; constraints[i].constraints = v0; constraints[i].weights = w0;
        }
    }
    std::vector<bsfm_point_constraints_t> point_constraints;
    if (use_point_constraints) {                                 // sfm.c:757-781
        if (!pt_constraints) { set_error("bsfm_run_sfm: use_point_constraints without points_constraints"); return BSFM_ERR_ARG; }
        point_constraints.resize(num_pts);
        for (int i = 0; i < num_pts; i++) {
            const double *q = pt_constraints[i].p;
            if (q[0] == 0.0 && q[1] == 0.0 && q[2] == 0.0) {
                point_constraints[i].constrained = 0;
                point_constraints[i].constraints[0] = point_constraints[i].constraints[1] = point_constraints[i].constraints[2] = 0.0;
                point_constraints[i].weight = 0.0;
            } else {
                point_constraints[i].constrained = 1;
                point_constraints[i].weight = pt_constraint_weight;
                point_constraints[i].constraints[0] = q[0]; point_constraints[i].constraints[1] = q[1]; point_constraints[i].constraints[2] = q[2];
            }
        }
    }

    bsfm_sfm_model_t model;
    model.est_focal_length = est_focal_length; model.undistort = undistort; model.explicit_camera_centers = explicit_camera_centers;
    model.f_scale = f_scale; model.k_scale = k_scale; model.R_init = R_init.data(); model.f_fixed = f_fixed.data();

    const char *verb_env = getenv("BSFM_BA_VERBOSE");
    const int verbosity = verb_env ? atoi(verb_env) : 3;          // VERBOSITY 3, MAX_ITERS 150 (sfm.c:814-815)
    int rc;
    if (fix_points)     // sfm.c:843-849: motion-only BA, the points come from init_pts and stay as they are
        rc = bsfm_sba_mot_levmar_model_ki(num_pts, num_cameras, ncons, vmask, params.data(), cnp, projections, nullptr, 2,
                                          &model, params.data() + num_camera_params, BSFM_BA_JAC_FD, 150, verbosity, opts, info,
                                          use_constraints, use_constraints ? constraints.data() : nullptr, init_camera_params);
    else
        rc = bsfm_sba_motstr_levmar_model_ki(num_pts, num_cameras, ncons, vmask, params.data(), cnp, 3, projections, nullptr, 2,
                                             &model, BSFM_BA_JAC_FD, 150, verbosity, opts, info,
                                             use_constraints, use_constraints ? constraints.data() : nullptr,
                                             use_point_constraints, use_point_constraints ? point_constraints.data() : nullptr,
                                             Vout, Sout, Uout, Wout, init_camera_params);
    if (rc < -1) {              // BSFM_ERR_*: nothing was solved; the caller's cameras get their scale fields back (they were set
        for (int j = 0; j < num_cameras; j++) { init_camera_params[j].f_scale = 1.0; init_camera_params[j].k_scale = 1.0; }   // to 0.001 / 5 above)
        return rc;
    }
    printf("[run_sfm] Number of iterations: %d\n", (int) info[5]);   // sfm.c:872-873
    printf("info[6] = %0.3f\n", info[6]);
    if (info_out) memcpy(info_out, info, sizeof info);

    // host-side rot_update for the unpacking (sfm.c:876-929); same arithmetic as the device version
    for (int j = 0; j < num_cameras; j++) {
        const double *dt = &params[(size_t) cnp * j + 0];
        const double *w = &params[(size_t) cnp * j + 3];
        int c;
        init_camera_params[j].t[0] = dt[0]; init_camera_params[j].t[1] = dt[1]; init_camera_params[j].t[2] = dt[2];
        {
            double *R = init_camera_params[j].R, Rnew[9];
            const double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
            if (theta != 0.0) {
                const double n0 = w[0] / theta, n1 = w[1] / theta, n2 = w[2] / theta;
                const double nx[9] = {0.0, -n2, n1, n2, 0.0, -n0, -n1, n0, 0.0};
                double nxsq[9], dR[9];
                for (int r = 0; r < 3; r++) for (int cc2 = 0; cc2 < 3; cc2++)
                    nxsq[3 * r + cc2] = nx[3 * r] * nx[cc2] + nx[3 * r + 1] * nx[3 + cc2] + nx[3 * r + 2] * nx[6 + cc2];
                const double sinth = sin(theta), costh = cos(theta);
                for (int q = 0; q < 9; q++) dR[q] = (((q % 4 == 0) ? 1.0 : 0.0) + nx[q] * sinth) + nxsq[q] * (1.0 - costh);
                for (int r = 0; r < 3; r++) for (int cc2 = 0; cc2 < 3; cc2++)
                    Rnew[3 * r + cc2] = dR[3 * r] * R[cc2] + dR[3 * r + 1] * R[3 + cc2] + dR[3 * r + 2] * R[6 + cc2];
                memcpy(R, Rnew, sizeof Rnew);
            }
        }
        if (est_focal_length) { c = 7; init_camera_params[j].f = params[(size_t) cnp * j + 6] / init_camera_params[j].f_scale; }
        else c = 6;
        if (undistort) {
            const double scale = init_camera_params[j].k_scale;
            init_camera_params[j].k[0] = params[(size_t) cnp * j + c] / scale;
            init_camera_params[j].k[1] = params[(size_t) cnp * j + c + 1] / scale;
        }
        init_camera_params[j].f_scale = 1.0;
        init_camera_params[j].k_scale = 1.0;
    }
    for (int i = 0; i < num_pts; i++)
        for (int q = 0; q < 3; q++) init_pts[i].p[q] = params[(size_t) num_camera_params + 3 * (size_t) i + q];
    return BSFM_OK;
}
