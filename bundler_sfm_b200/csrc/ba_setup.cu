// ba_setup.cu -- setup of a BA call (ba_setup.h): device memory pool, visibility (mask or CRS) -> CRS and camera-major permutation,
// Schur structure, and the kernels that build them.
#include "ba_setup.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <climits>
#include <cstdlib>
#include <map>
#include <mutex>

namespace bsfm {
namespace ba {

// structure-building kernels: vmask -> CRS, camera-major permutation, Schur tuples
__global__ void vmask_count_kernel(const char *vmask, int n, int m, int *row_count)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    int c = 0;
    for (int j = lane; j < m; j += 32) c += vmask[(size_t) i * m + j] != 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if (lane == 0) row_count[i] = c;
}

__global__ void vmask_fill_kernel(const char *vmask, int n, int m, const int *rowptr, int *obs_cam, int *obs_pt)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    int pos = rowptr[i];
    for (int j0 = 0; j0 < m; j0 += 32) {
        const int j = j0 + lane;
        const bool v = j < m && vmask[(size_t) i * m + j] != 0;
        const unsigned ball = __ballot_sync(0xffffffffu, v);
        if (v) {
            const int q = pos + __popc(ball & ((1u << lane) - 1u));
            obs_cam[q] = j; obs_pt[q] = i;
        }
        pos += __popc(ball);
    }
}

// obs_pt from the CRS row pointers (the host-scanned visibility mask below): one warp per point
__global__ void csr_rows_kernel(const int *rowptr, int n, int *obs_pt)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    for (int q = rowptr[i] + lane; q < rowptr[i + 1]; q += 32) obs_pt[q] = i;
}

// Why a caller's CRS is refused; for one point the lowest code is reported
enum CrsFault { CRS_FIRST_PTR = 1, CRS_LAST_PTR, CRS_PTR_RANGE, CRS_PTR_DECREASES, CRS_CAM_RANGE, CRS_CAM_ORDER };

// A caller's CRS, checked before anything else reads it, one warp per point; obs_pt is filled on the way.  The lowest
// faulty point and its lowest fault go to *verdict as (point << 3 | fault) (left at ~0 when the CRS is sound).  Every
// index is bounded before it is dereferenced: point i < n reads rowptr[i] and rowptr[i + 1] (n + 1 entries), and
// obs_cam / obs_pt are touched only at q in [p0, p1) after 0 <= p0 <= p1 <= nvis has been established.
__global__ void crs_check_kernel(const int *rowptr, const int *obs_cam, int n, int m, int nvis, int *obs_pt,
                                 unsigned long long *verdict)
{
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const int p0 = rowptr[i], p1 = rowptr[i + 1];
    int fault = 0;
    if (i == 0 && p0 != 0) fault = CRS_FIRST_PTR;
    else if (i == n - 1 && p1 != nvis) fault = CRS_LAST_PTR;
    else if (p0 < 0 || p1 > nvis) fault = CRS_PTR_RANGE;
    else if (p1 < p0) fault = CRS_PTR_DECREASES;
    if (fault) {
        if (lane == 0) atomicMin(verdict, ((unsigned long long) i << 3) | fault);
        return;
    }
    for (int q = p0 + lane; q < p1; q += 32) {
        const int c = obs_cam[q];
        fault = (c < 0 || c >= m) ? CRS_CAM_RANGE : (q > p0 && obs_cam[q - 1] >= c) ? CRS_CAM_ORDER : 0;
        if (fault) atomicMin(verdict, ((unsigned long long) i << 3) | fault);
        obs_pt[q] = i;
    }
}

__global__ void iota_kernel(int *v, int count)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < count) v[q] = q;
}

// cam_ptr[j] = first position of camera j in the camera-sorted key array
__global__ void cam_ptr_kernel(const int *sorted_cam, int nvis, int m, int *cam_ptr)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > m) return;
    int lo = 0, hi = nvis;   // first position with cam >= j
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sorted_cam[mid] < j) lo = mid + 1; else hi = mid;
    }
    cam_ptr[j] = lo;
}

// tuples of point i: all (a <= b) pairs of its observations restricted to cameras >= mcon
__global__ void tuple_count_kernel(int n, int mcon, const int *rowptr, const int *obs_cam, int *tuple_count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int L = 0;
    for (int o = rowptr[i]; o < rowptr[i + 1]; o++) L += obs_cam[o] >= mcon;
    tuple_count[i] = L * (L + 1) / 2;
}

__global__ void tuple_fill_kernel(int n, int m, int mcon, const int *rowptr, const int *obs_cam, const int *tuple_off,
                                  uint32_t *keys, int2 *vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int pos = tuple_off[i];
    const int r0 = rowptr[i], r1 = rowptr[i + 1];
    for (int a = r0; a < r1; a++) {
        const int ja = obs_cam[a];
        if (ja < mcon) continue;
        for (int b = a; b < r1; b++) {
            const int jb = obs_cam[b];   // ascending camera order inside a row => ja <= jb
            keys[pos] = (uint32_t) ja * (uint32_t) m + (uint32_t) jb;
            vals[pos] = make_int2(a, b);
            pos++;
        }
    }
}

// sorted (obs_a, obs_b) -> (obs_a, obs_b, point, 0)
__global__ void tuple_expand_kernel(const int2 *in, const int *obs_pt, int4 *out, int count)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < count) { const int2 v = in[q]; out[q] = make_int4(v.x, v.y, obs_pt[v.x], 0); }
}

__global__ void chunk_count_kernel(const int *blk_cnt, int nblocks, int *chunk_cnt)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nblocks) chunk_cnt[b] = (blk_cnt[b] + SCHUR_CHUNK - 1) / SCHUR_CHUNK;
    else if (b == nblocks) chunk_cnt[b] = 0;
}

namespace {
// Device blocks are recycled across calls (RunSFM_SBA calls run_sfm once per outlier round on a problem of
// nearly the same size, src/Bundle.cpp:586-913): cudaMalloc/cudaFree cost tens of microseconds each and a solve of the
// 50-camera configuration only takes milliseconds.  Blocks return to a per-process pool when a call ends.
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
BlockPool g_pool;
}  // namespace

thread_local UploadTally t_uploads;
void count_upload(const void *src, size_t bytes)
{
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, src) != cudaSuccess) { cudaGetLastError(); return; }
    if (pa.type != cudaMemoryTypeHost && pa.type != cudaMemoryTypeUnregistered) return;
    t_uploads.bytes += (long long) bytes;
    t_uploads.largest = std::max(t_uploads.largest, (long long) bytes);
}

DeviceArena::~DeviceArena()
{
    if (!blocks.empty()) cudaStreamSynchronize(st);
    for (auto &b : blocks) g_pool.put(b.first, b.second);
}

int DeviceArena::alloc_bytes(void **out, size_t bytes)
{
    if (blocks.empty()) { int dev = 0; BSFM_CUDA_TRY(cudaGetDevice(&dev)); g_pool.bind_device(dev); }
    bytes = (bytes + 255) & ~(size_t) 255;
    size_t cap = bytes;
    void *p = g_pool.get(bytes, &cap);
    if (!p) {
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString(e)); return BSFM_ERR_CUDA; }
        cap = bytes;
    }
    blocks.push_back({p, cap});
    *out = p;
    return BSFM_OK;
}

namespace {
const char *crs_fault_text(int fault)
{
    switch (fault) {
    case CRS_FIRST_PTR: return "vis_ptr[0] != 0";
    case CRS_LAST_PTR: return "vis_ptr[num_pts] != nvis";
    case CRS_PTR_RANGE: return "vis_ptr outside [0, nvis]";
    case CRS_PTR_DECREASES: return "vis_ptr decreases";
    case CRS_CAM_RANGE: return "camera index outside [0, num_cameras)";
    default: return "cameras not strictly ascending";
    }
}
}  // namespace

// Visibility (idxij, sba_levmar.c:652-663) from one of three sources:
//   1. a dense mask scanned on the device: count, cub scan, one sync for nvis, fill of obs_cam and obs_pt;
//   2. a host-resident dense mask scanned on the host (host_scan_vmask, behind BSFM_BA_MASK_HOST_MIN);
//   3. the caller's CRS, checked on the device (crs_check_kernel) with one sync for the verdict before anything reads it.
// Sources 2 and 3 share the CRS upload, and all three the camera-major tail, so the same visibility gives the same arrays
// whichever source it came from.
int build_visibility(const VisSource &src, int n, int m, cudaStream_t st, DeviceArena &D, Visibility &V)
{
    // host-resident masks of at least BSFM_BA_MASK_HOST_MIN bytes are scanned on the host and only their CRS form is uploaded
    // (host_scan_vmask, common.cpp).  OFF by default: at config 3 it cuts the H2D bytes per solve from 560 to 75 MB, but the scan
    // of the 500 MB mask costs host time, and whether it beats the PCIe copy from pinned memory depends on the host.
    static const size_t host_scan_min = []() { const char *e = getenv("BSFM_BA_MASK_HOST_MIN"); return e ? (size_t) atoll(e) : ~(size_t) 0; }();
    bool host_mask = false;
    if (src.vmask && (size_t) n * m >= host_scan_min) {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, src.vmask) == cudaSuccess) host_mask = (pa.type == cudaMemoryTypeHost || pa.type == cudaMemoryTypeUnregistered);
        else cudaGetLastError();
    }
    if (src.vmask && !host_mask) {   // source 1
        char *d_vmask;
        int *d_rowcnt;
        TRY(D.alloc(&d_rowcnt, (size_t) n + 1));
        TRY(D.alloc(&V.rowptr, (size_t) n + 1));
        TRY(D.upload(&d_vmask, src.vmask, (size_t) n * m));   // host or device pointer (UVA)
        BSFM_CUDA_TRY(cudaMemsetAsync(d_rowcnt, 0, ((size_t) n + 1) * sizeof(int), st));
        vmask_count_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(d_vmask, n, m, d_rowcnt);
        BSFM_KERNEL_CHECK();
        TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, d_rowcnt, V.rowptr, n + 1, st); }));
        BSFM_CUDA_TRY(cudaMemcpyAsync(&V.nvis, V.rowptr + n, sizeof(int), cudaMemcpyDeviceToHost, st));
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));
        if (V.nvis <= 0) return BSFM_OK;
        TRY(D.alloc(&V.obs_cam, (size_t) V.nvis)); TRY(D.alloc(&V.obs_pt, (size_t) V.nvis));
        vmask_fill_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(d_vmask, n, m, V.rowptr, V.obs_cam, V.obs_pt);
        BSFM_KERNEL_CHECK();
    } else if (src.ours) {           // device CRS written by the library: used where it is, obs_pt from the row pointers
        V.nvis = src.nvis;
        V.rowptr = const_cast<int *>(src.vis_ptr);
        if (V.nvis > 0) {
            V.obs_cam = const_cast<int *>(src.vis_cam);
            TRY(D.alloc(&V.obs_pt, (size_t) V.nvis));
            csr_rows_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(V.rowptr, n, V.obs_pt);
            BSFM_KERNEL_CHECK();
        }
    } else {                         // sources 2 and 3: CRS arrays in host or device memory
        std::vector<int> h_rowptr, h_obs_cam;
        const int *rowptr = src.vis_ptr, *obs_cam = src.vis_cam;
        if (host_mask) {
            host_scan_vmask(src.vmask, n, m, h_rowptr, h_obs_cam);
            rowptr = h_rowptr.data(); obs_cam = h_obs_cam.data();
            V.nvis = h_rowptr[n];
        } else {
            if (src.nvis < 0 || src.nvis > INT_MAX / 2) {   // the solver counts 2 * nvis measurements in an int
                set_error("malformed visibility (CRS): nvis = %d is outside [0, %d]", src.nvis, INT_MAX / 2);
                return BSFM_ERR_ARG;
            }
            V.nvis = src.nvis;
        }
        TRY(D.alloc(&V.rowptr, (size_t) n + 1));
        note_upload(rowptr, ((size_t) n + 1) * sizeof(int));
        BSFM_CUDA_TRY(cudaMemcpyAsync(V.rowptr, rowptr, ((size_t) n + 1) * sizeof(int), cudaMemcpyDefault, st));
        if (V.nvis > 0) {
            TRY(D.alloc(&V.obs_cam, (size_t) V.nvis)); TRY(D.alloc(&V.obs_pt, (size_t) V.nvis));
            note_upload(obs_cam, (size_t) V.nvis * sizeof(int));
            BSFM_CUDA_TRY(cudaMemcpyAsync(V.obs_cam, obs_cam, (size_t) V.nvis * sizeof(int), cudaMemcpyDefault, st));
        }
        if (host_mask) {
            if (V.nvis > 0) {
                csr_rows_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(V.rowptr, n, V.obs_pt);
                BSFM_KERNEL_CHECK();
            }
        } else {
            unsigned long long *d_verdict, verdict = 0;
            TRY(D.alloc(&d_verdict, 1));
            BSFM_CUDA_TRY(cudaMemsetAsync(d_verdict, 0xff, sizeof(unsigned long long), st));
            crs_check_kernel<<<(n * 32 + 255) / 256, 256, 0, st>>>(V.rowptr, V.obs_cam, n, m, V.nvis, V.obs_pt, d_verdict);
            BSFM_KERNEL_CHECK();
            BSFM_CUDA_TRY(cudaMemcpyAsync(&verdict, d_verdict, sizeof verdict, cudaMemcpyDeviceToHost, st));
            BSFM_CUDA_TRY(cudaStreamSynchronize(st));
            if (verdict != ~0ULL) {
                set_error("malformed visibility (CRS) at point %d: %s", (int) (verdict >> 3), crs_fault_text((int) (verdict & 7)));
                return BSFM_ERR_ARG;
            }
        }
    }
    // the shared tail: camera-major permutation, a stable sort of observation ids by camera.  The int keys sort as they
    // are: cub's signed-key transform flips bit 31 only, outside the sorted bits [0, bits).
    const int nvis = V.nvis;
    if (nvis <= 0) return BSFM_OK;
    int *d_iota, *d_cam_sorted;
    TRY(D.alloc(&V.cam_ptr, (size_t) m + 1)); TRY(D.alloc(&V.cam_obs, (size_t) nvis)); TRY(D.alloc(&d_iota, (size_t) nvis));
    TRY(D.alloc(&d_cam_sorted, (size_t) nvis));
    iota_kernel<<<(nvis + 255) / 256, 256, 0, st>>>(d_iota, nvis);
    BSFM_KERNEL_CHECK();
    int bits = 1; while ((1LL << bits) < m) bits++;
    TRY(D.cub(3, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, V.obs_cam, d_cam_sorted, d_iota, V.cam_obs, nvis, 0, bits, st); }));
    cam_ptr_kernel<<<(m + 1 + 255) / 256, 256, 0, st>>>(d_cam_sorted, nvis, m, V.cam_ptr);
    BSFM_KERNEL_CHECK();
    return BSFM_OK;
}

// Schur structure: (obs_a, obs_b) tuples of every point, sorted by block key j*m+k (stable => ascending point)
int build_schur_structure(Problem &P, cudaStream_t st, DeviceArena &D)
{
    const int n = P.n, m = P.m, mcon = P.mcon;
    int *d_tcnt, *d_toff;
    TRY(D.alloc(&d_tcnt, (size_t) n + 1)); TRY(D.alloc(&d_toff, (size_t) n + 1));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_tcnt, 0, ((size_t) n + 1) * sizeof(int), st));
    tuple_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, mcon, P.rowptr, P.obs_cam, d_tcnt);
    BSFM_KERNEL_CHECK();
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, d_tcnt, d_toff, n + 1, st); }));
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
    tuple_fill_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, m, mcon, P.rowptr, P.obs_cam, d_toff, d_tkey_a, (int2 *) d_tval_a);
    BSFM_KERNEL_CHECK();
    int bits = 1; while ((1LL << bits) < (long long) m * m) bits++;
    TRY(D.cub(3, [&](void *t, size_t &b) { return cub::DeviceRadixSort::SortPairs(t, b, d_tkey_a, d_tkey_b, d_tval_a, d_tval_b, ntuples, 0, bits, st); }));
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceRunLengthEncode::Encode(t, b, d_tkey_b, d_blk_key, d_blk_cnt, d_nruns, ntuples, st); }));
    int nblocks = 0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(&nblocks, d_nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_blk_cnt + nblocks, 0, sizeof(int), st));
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, d_blk_cnt, d_blk_start, nblocks + 1, st); }));
    // chunk list (SCHUR_CHUNK tuples per partial-sum warp) + (obs_a, obs_b, point) tuples
    int *d_chunk_cnt, *d_chunk_off;
    int4 *d_tuples4;
    TRY(D.alloc(&d_chunk_cnt, (size_t) nblocks + 1)); TRY(D.alloc(&d_chunk_off, (size_t) nblocks + 1));
    TRY(D.alloc(&d_tuples4, (size_t) ntuples));
    chunk_count_kernel<<<(nblocks + 1 + 255) / 256, 256, 0, st>>>(d_blk_cnt, nblocks, d_chunk_cnt);
    BSFM_KERNEL_CHECK();
    TRY(D.cub(2, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, d_chunk_cnt, d_chunk_off, nblocks + 1, st); }));
    tuple_expand_kernel<<<(ntuples + 255) / 256, 256, 0, st>>>((const int2 *) d_tval_b, P.obs_pt, d_tuples4, ntuples);
    BSFM_KERNEL_CHECK();
    int nchunks = 0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(&nchunks, d_chunk_off + nblocks, sizeof(int), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    P.nblocks = nblocks; P.blk_key = d_blk_key; P.blk_start = d_blk_start; P.tuples = d_tuples4;
    P.nchunks = nchunks; P.chunk_off = d_chunk_off;
    TRY(D.alloc(&P.schur_part, (size_t) nchunks * SCHUR_PART_STRIDE));
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm
