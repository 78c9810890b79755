// match_api.cu -- host side of the MATCH path behind the C ABI of include/bsfm_b200.h.
// Mirrors the loop structure of src/KeyMatchFull.cpp:105-151 (i ascending, j ascending inside the
// window) and the MatchKeys contract of src/keys2a.cpp:347-424.  No CPU fallback.
#include "common.h"
#include "match_kernels.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <algorithm>
#include <atomic>
#include <climits>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace bsfm {
namespace match {
// kernels (match_kernels.cu)
__global__ void raw_norm_kernel(const uint8_t *, int64_t, int32_t *, int32_t *);
__global__ void prep_kernel(const uint8_t *, const int64_t *, const int32_t *, const int32_t *, const int32_t *, const int32_t *, uint8_t *, int32_t *, int32_t *, int64_t, int64_t, int64_t);
__global__ void match_dp4a_kernel(MatchParams);
__global__ void match_tc_kernel(MatchParams);
__global__ void match_tc_bound_kernel(MatchParams);
__global__ void match_tc_quad_kernel(MatchParams);
__global__ void match_tc_pair_kernel(MatchParams);
__global__ void match_verify_kernel(MatchParams, int);
__global__ void match_fullscan_kernel(MatchParams, int);
__global__ void match_finalize_kernel(const uint32_t *, const int32_t *, int, const RunImage *, int, int,
                                      const int32_t *, const int32_t *, const int32_t *, int32_t *, int32_t *);
}  // namespace match
}  // namespace bsfm

using namespace bsfm;
using namespace bsfm::match;

struct bsfm_keydb {
    int N = 0;
    int device = 0;
    int num_sms = 0;
    std::vector<int64_t> key_off;   // N+1
    std::vector<int32_t> doff;      // N+1 device row offsets (multiples of 256); a sharded build leaves gaps between groups
    std::vector<int32_t> img_rows;  // N padded row counts
    int64_t drows = 0;
    uint8_t *d_keys_sw = nullptr;
    int32_t *d_norms = nullptr;
    int32_t *d_perm = nullptr;
    int32_t *d_tile_img = nullptr;
    int32_t *d_img_doff = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // result of the last run
    int64_t shard_pairs = 0;
    int64_t total_matches = 0;
    int32_t *d_pair_counts = nullptr;
    int64_t pair_cap = 0;
    int32_t *d_matches = nullptr;   // [match_cap][2]
    int64_t match_cap = 0;
    float ms[3] = {0, 0, 0};
    int launches = 0;
    int64_t cand_rows = 0, hard_rows = 0;   // statistics of the last run (tensor-core kernel)
    // scratch reused across runs
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
    // table gathered from all ranks (bsfm_match_allgather)
    int32_t *d_gather_counts = nullptr, *d_gather_matches = nullptr;
    int64_t gather_pairs = 0, gather_matches = 0, gather_pair_cap = 0, gather_match_cap = 0;
};

// ---- NCCL, bound at run time (dlopen): libbsfm_b200.so has no link-time dependency on it, single-GPU users never load
// it, and inside a torch process the already loaded libnccl.so.2 is the one that answers ------------------------------
#include <dlfcn.h>
#include <nccl.h>
namespace {
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
NcclApi &nccl_api()
{
    static NcclApi api = []() {
        NcclApi a;
        for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
            a.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (a.handle) break;
        }
        if (!a.handle) return a;
        a.GetUniqueId = (decltype(a.GetUniqueId)) dlsym(a.handle, "ncclGetUniqueId");
        a.CommInitRank = (decltype(a.CommInitRank)) dlsym(a.handle, "ncclCommInitRank");
        a.CommDestroy = (decltype(a.CommDestroy)) dlsym(a.handle, "ncclCommDestroy");
        a.AllGather = (decltype(a.AllGather)) dlsym(a.handle, "ncclAllGather");
        a.Broadcast = (decltype(a.Broadcast)) dlsym(a.handle, "ncclBroadcast");
        a.GroupStart = (decltype(a.GroupStart)) dlsym(a.handle, "ncclGroupStart");
        a.GroupEnd = (decltype(a.GroupEnd)) dlsym(a.handle, "ncclGroupEnd");
        a.GetErrorString = (decltype(a.GetErrorString)) dlsym(a.handle, "ncclGetErrorString");
        a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.Broadcast && a.GroupStart && a.GroupEnd && a.GetErrorString;
        return a;
    }();
    return api;
}
}  // namespace
#define BSFM_NCCL_TRY(expr)                                                                                      \
    do {                                                                                                          \
        ncclResult_t r__ = (expr);                                                                                \
        if (r__ != ncclSuccess) {                                                                                 \
            set_error("%s failed: %s (%s:%d)", #expr, nccl_api().GetErrorString(r__), __FILE__, __LINE__);        \
            return BSFM_ERR_CUDA;                                                                                 \
        }                                                                                                         \
    } while (0)

struct bsfm_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
};

static int env_int(const char *name, int dflt)
{
    const char *v = getenv(name);
    return v ? atoi(v) : dflt;
}

// `comm` != null: cooperative build -- the images are split into `world` contiguous groups of (nearly) equal key count,
// this rank uploads / sorts / swizzles only ITS group into its chunk of the device layout (chunks of equal size, so the
// prepared rows are exchanged by ONE in-place ncclAllGather per array over NVLink) and ends with the complete database.
static int keydb_build(bsfm_keydb *db, const uint8_t *keys, bool keys_on_device, const int64_t *key_off, int N, const bsfm_comm *comm = nullptr)
{
    int rc = require_device();
    if (rc != BSFM_OK) return rc;
    if (N < 0 || (N > 0 && (!key_off || key_off[0] != 0))) {
        set_error("bsfm_keydb_create: bad arguments (N=%d)", N);
        return BSFM_ERR_ARG;
    }
    db->N = N;
    BSFM_CUDA_TRY(cudaGetDevice(&db->device));
    cudaDeviceProp prop;
    BSFM_CUDA_TRY(cudaGetDeviceProperties(&prop, db->device));
    db->num_sms = prop.multiProcessorCount;
    db->key_off.assign(key_off, key_off + N + 1);
    db->doff.resize(N + 1);
    for (int i = 0; i < N; i++)
        if (key_off[i + 1] < key_off[i]) { set_error("bsfm_keydb_create: key_off not monotone at %d", i); return BSFM_ERR_ARG; }
    const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
    // image groups [gb[g], gb[g+1]) of (nearly) equal key count; one group = everything when not sharded
    std::vector<int> gb((size_t) world + 1, N);
    gb[0] = 0;
    {
        const int64_t total = key_off[N];
        int g = 1;
        for (int i = 0; i < N && g < world; i++)
            while (g < world && key_off[i + 1] * world >= total * g) gb[(size_t) g++] = i + 1;
    }
    auto padded = [&](int i) { return (key_off[i + 1] - key_off[i] + IMG_PAD - 1) / IMG_PAD * IMG_PAD; };
    int64_t chunk_rows = 0;
    for (int g = 0; g < world; g++) {
        int64_t rows = 0;
        for (int i = gb[(size_t) g]; i < gb[(size_t) g + 1]; i++) rows += padded(i);
        chunk_rows = std::max(chunk_rows, rows);
    }
    if (chunk_rows * world > (int64_t) INT_MAX - 1024) { set_error("bsfm_keydb_create: more than 2^31 descriptor rows"); return BSFM_ERR_ARG; }
    for (int g = 0; g < world; g++) {
        int64_t r = (int64_t) g * chunk_rows;
        for (int i = gb[(size_t) g]; i < gb[(size_t) g + 1]; i++) { db->doff[i] = (int32_t) r; r += padded(i); }
    }
    db->doff[N] = (int32_t) (chunk_rows * world);
    db->drows = chunk_rows * world + IMG_PAD;   // one spare padded tile so any 256-row read stays in bounds
    const int64_t ntiles = db->drows / TILE_Q;
    std::vector<int32_t> tile_img((size_t) ntiles, -1);
    for (int i = 0; i < N; i++)
        for (int64_t t = db->doff[i] / TILE_Q; t < (db->doff[i] + padded(i)) / TILE_Q; t++) tile_img[(size_t) t] = i;
    db->img_rows.resize(N);
    for (int i = 0; i < N; i++) db->img_rows[(size_t) i] = (int32_t) padded(i);

    BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&db->stream, cudaStreamNonBlocking));
    for (int e = 0; e < 4; e++) BSFM_CUDA_TRY(cudaEventCreate(&db->ev[e]));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_keys_sw, (size_t) db->drows * DESC_BYTES));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_norms, (size_t) db->drows * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_perm, (size_t) db->drows * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_tile_img, (size_t) ntiles * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_img_doff, (size_t) (N + 1) * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_tile_img, tile_img.data(), (size_t) ntiles * sizeof(int32_t), cudaMemcpyHostToDevice, db->stream));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_img_doff, db->doff.data(), (size_t) (N + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, db->stream));

    // this rank's group of images: keys [kb, ke), images [ib, ie), device rows [row_b, row_e)
    const int ib = gb[(size_t) rank], ie = gb[(size_t) rank + 1];
    const int64_t kb = key_off[ib], ke = key_off[ie];
    const int64_t total_keys = ke - kb;
    const int64_t row_b = (int64_t) rank * chunk_rows, row_e = row_b + chunk_rows;
    uint8_t *d_raw = nullptr;
    int64_t *d_key_off = nullptr;
    // temporaries are released on every exit path (an early BSFM_CUDA_TRY return used to leak them)
    struct Temps {
        std::vector<void *> ptrs;
        ~Temps() { for (void *q : ptrs) cudaFree(q); }
        void own(void *q) { if (q) ptrs.push_back(q); }
    } temps;
    BSFM_CUDA_TRY(cudaMalloc(&d_key_off, (size_t) (N + 1) * sizeof(int64_t)));
    temps.own(d_key_off);
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_key_off, key_off, (size_t) (N + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, db->stream));
    if (keys_on_device) {
        d_raw = const_cast<uint8_t *>(keys) + (size_t) kb * DESC_BYTES;
    } else if (total_keys > 0) {
        BSFM_CUDA_TRY(cudaMalloc(&d_raw, (size_t) total_keys * DESC_BYTES));
        temps.own(d_raw);
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_raw, keys + (size_t) kb * DESC_BYTES, (size_t) total_keys * DESC_BYTES, cudaMemcpyHostToDevice, db->stream));
    }
    // per-image stable sort of the keys by squared norm (the tensor-core epilogue relies on norm-sorted chunks)
    int32_t *d_nraw = nullptr, *d_nsorted = nullptr, *d_iota = nullptr, *d_src = nullptr, *d_seg = nullptr;
    void *d_tmp = nullptr;
    if (key_off[N] > (int64_t) INT_MAX - 1) { set_error("bsfm_keydb_create: more than 2^31 keys"); return BSFM_ERR_ARG; }
    const size_t nk = (size_t) std::max<int64_t>(total_keys, 1);
    const int nseg = ie - ib;
    BSFM_CUDA_TRY(cudaMalloc(&d_nraw, nk * 4)); temps.own(d_nraw);
    BSFM_CUDA_TRY(cudaMalloc(&d_nsorted, nk * 4)); temps.own(d_nsorted);
    BSFM_CUDA_TRY(cudaMalloc(&d_iota, nk * 4)); temps.own(d_iota);
    BSFM_CUDA_TRY(cudaMalloc(&d_src, nk * 4)); temps.own(d_src);
    BSFM_CUDA_TRY(cudaMalloc(&d_seg, (size_t) (nseg + 1) * 4)); temps.own(d_seg);
    if (total_keys > 0) {
        std::vector<int32_t> seg((size_t) nseg + 1);
        for (int i = 0; i <= nseg; i++) seg[(size_t) i] = (int32_t) (key_off[ib + i] - kb);
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_seg, seg.data(), (size_t) (nseg + 1) * 4, cudaMemcpyHostToDevice, db->stream));
        raw_norm_kernel<<<(unsigned) ((total_keys + 7) / 8), 256, 0, db->stream>>>(d_raw, total_keys, d_nraw, d_iota);
        BSFM_KERNEL_CHECK();
        size_t tb = 0;
        cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, d_nraw, d_nsorted, d_iota, d_src, (int) total_keys, nseg, d_seg, d_seg + 1, db->stream);
        BSFM_CUDA_TRY(cudaMalloc(&d_tmp, std::max<size_t>(tb, 1)));
        temps.own(d_tmp);
        cub::DeviceSegmentedSort::StableSortPairs(d_tmp, tb, d_nraw, d_nsorted, d_iota, d_src, (int) total_keys, nseg, d_seg, d_seg + 1, db->stream);
        count_launch(3);
        BSFM_CUDA_TRY(cudaGetLastError());
        BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));   // seg[] is a host temporary
    }
    {
        const int warps_per_block = 8;
        // own chunk, then the spare tile behind the last chunk (padding rows; every rank writes its own copy)
        const int64_t spans[2][2] = {{row_b, row_e}, {chunk_rows * world, db->drows}};
        for (int q = 0; q < 2; q++) {
            const int64_t rows = spans[q][1] - spans[q][0];
            if (rows <= 0) continue;
            const int64_t blocks = (rows + warps_per_block - 1) / warps_per_block;
            prep_kernel<<<(unsigned) blocks, warps_per_block * 32, 0, db->stream>>>(d_raw, d_key_off, db->d_img_doff, db->d_tile_img, d_src, d_nsorted,
                                                                                     db->d_keys_sw, db->d_norms, db->d_perm, spans[q][0], spans[q][1], kb);
            BSFM_KERNEL_CHECK();
        }
    }
    if (comm && world > 1) {
        NcclApi &nc = nccl_api();
        BSFM_NCCL_TRY(nc.GroupStart());
        BSFM_NCCL_TRY(nc.AllGather(db->d_keys_sw + (size_t) row_b * DESC_BYTES, db->d_keys_sw, (size_t) chunk_rows * DESC_BYTES, ncclUint8, comm->comm, db->stream));
        BSFM_NCCL_TRY(nc.AllGather(db->d_norms + row_b, db->d_norms, (size_t) chunk_rows, ncclInt32, comm->comm, db->stream));
        BSFM_NCCL_TRY(nc.AllGather(db->d_perm + row_b, db->d_perm, (size_t) chunk_rows, ncclInt32, comm->comm, db->stream));
        BSFM_NCCL_TRY(nc.GroupEnd());
    }
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    return BSFM_OK;
}

static int start_image(int i, int window_radius) { return (window_radius > 0) ? std::max(i - window_radius, 0) : 0; }

static int ensure_scratch(bsfm_keydb *db, size_t bytes)
{
    if (db->scratch_bytes >= bytes) return BSFM_OK;
    if (db->scratch) cudaFree(db->scratch);
    db->scratch = nullptr; db->scratch_bytes = 0;
    BSFM_CUDA_TRY(cudaMalloc(&db->scratch, bytes));
    db->scratch_bytes = bytes;
    return BSFM_OK;
}

static int grow_matches(bsfm_keydb *db, int64_t need)
{
    if (db->match_cap >= need) return BSFM_OK;
    int64_t cap = std::max<int64_t>(need, std::max<int64_t>(db->match_cap * 2, 1 << 16));
    int32_t *p = nullptr;
    BSFM_CUDA_TRY(cudaMalloc(&p, (size_t) cap * 2 * sizeof(int32_t)));
    if (db->d_matches && db->total_matches > 0)
        BSFM_CUDA_TRY(cudaMemcpyAsync(p, db->d_matches, (size_t) db->total_matches * 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    if (db->d_matches) cudaFree(db->d_matches);
    db->d_matches = p;
    db->match_cap = cap;
    return BSFM_OK;
}

static int64_t match_run_impl(bsfm_keydb *db, int img_begin, int img_end, int window_radius, double ratio, int test_mode = 0)
{
    clear_error();
    if (!db) { set_error("bsfm_match_run: null db"); return BSFM_ERR_ARG; }
    if (img_begin < 0 || img_end > db->N || img_begin > img_end) {
        set_error("bsfm_match_run: image range [%d,%d) outside [0,%d)", img_begin, img_end, db->N);
        return BSFM_ERR_ARG;
    }
    BSFM_CUDA_TRY(cudaSetDevice(db->device));
    const int kernel_sel = env_int("BSFM_MATCH_KERNEL", BSFM_MATCH_KERNEL_TC);
    const long long launches0 = g_kernel_launches.load();

    // ---- run tables: KeyMatchFull.cpp:105-123 ------------------------------------------------
    std::vector<RunImage> run;
    int64_t npairs = 0;
    int64_t nunits = 0;
    for (int i = img_begin; i < img_end; i++) {
        const int s = start_image(i, window_radius);
        const int64_t n_i = db->key_off[i + 1] - db->key_off[i];
        const int units = (db->doff[i] - db->doff[s]) / TILE_Q;
        if (n_i > 0 && units > 0) {
            RunImage R;
            R.img = i; R.n = (int32_t) n_i; R.db_row0 = db->doff[i];
            R.ntiles_db = db->img_rows[(size_t) i] / TILE_DB;
            R.atile0 = db->doff[s] / TILE_Q; R.start_img = s;
            R.unit0 = (int32_t) nunits; R.nunits = units; R.pair0 = npairs;
            if (nunits + units > (int64_t) INT_MAX / 2) { set_error("bsfm_match_run: shard too large (work units overflow)"); return BSFM_ERR_ARG; }
            run.push_back(R);
            nunits += units;
        }
        npairs += i - s;
    }
    db->shard_pairs = npairs;
    db->total_matches = 0;
    db->cand_rows = db->hard_rows = 0;
    db->ms[0] = db->ms[1] = db->ms[2] = 0;

    if (npairs > db->pair_cap) {
        if (db->d_pair_counts) cudaFree(db->d_pair_counts);
        db->d_pair_counts = nullptr; db->pair_cap = 0;
        BSFM_CUDA_TRY(cudaMalloc(&db->d_pair_counts, (size_t) std::max<int64_t>(npairs, 1) * sizeof(int32_t)));
        db->pair_cap = std::max<int64_t>(npairs, 1);
    }
    BSFM_CUDA_TRY(cudaEventRecord(db->ev[0], db->stream));
    if (npairs > 0) BSFM_CUDA_TRY(cudaMemsetAsync(db->d_pair_counts, 0, (size_t) npairs * sizeof(int32_t), db->stream));
    if (run.empty()) {
        BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
        db->launches = 0;
        return 0;
    }

    const int K = (int) run.size();
    RunImage *d_run = nullptr;
    BSFM_CUDA_TRY(cudaMalloc(&d_run, (size_t) K * sizeof(RunImage)));
    struct RunGuard { RunImage *&q; ~RunGuard() { if (q) cudaFree(q); q = nullptr; } } run_guard{d_run};   // freed on every exit path
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_run, run.data(), (size_t) K * sizeof(RunImage), cudaMemcpyHostToDevice, db->stream));

    // ---- chunked launches ---------------------------------------------------------------------
    const int64_t chunk_slots = std::max(1, env_int("BSFM_MATCH_CHUNK_MSLOTS", 32)) * (int64_t) (1 << 20);
    const int64_t chunk_units = std::max<int64_t>(1, chunk_slots / TILE_Q);
    int64_t biggest_img = 1;
    for (const RunImage &R : run) biggest_img = std::max<int64_t>(biggest_img, R.nunits);
    const int64_t max_units = std::min<int64_t>(std::max(chunk_units, biggest_img), nunits);
    const int64_t cap = max_units * TILE_Q;   // worst case: every query row is a candidate / match

    // scratch carve-up
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t *) nullptr, (uint32_t *) nullptr,
                                    (const int32_t *) nullptr, (int32_t *) nullptr, (int) std::min<int64_t>(cap, INT_MAX), 0, 32, db->stream);
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t) 255; return o; };
    const size_t o_cand = carve((size_t) cap * 7 * sizeof(int32_t));
    const size_t o_hard = carve((size_t) cap * 2 * sizeof(int32_t));
    const size_t o_slot_a = carve((size_t) cap * sizeof(uint32_t));
    const size_t o_slot_b = carve((size_t) cap * sizeof(uint32_t));
    const size_t o_idx_a = carve((size_t) cap * sizeof(int32_t));
    const size_t o_idx_b = carve((size_t) cap * sizeof(int32_t));
    const size_t o_cnt = carve(64);
    const size_t o_cub = carve(cub_bytes);
    int rc = ensure_scratch(db, off);
    if (rc != BSFM_OK) { return rc; }
    uint8_t *S = (uint8_t *) db->scratch;

    MatchParams P;
    P.keys_sw = db->d_keys_sw; P.norms = db->d_norms; P.run_imgs = d_run; P.num_run_imgs = K;
    P.perm = db->d_perm; P.tile_img = db->d_tile_img; P.img_doff = db->d_img_doff;
    // test mode 1 (keys.cpp:786): final decisions evaluate sqrt(d0 / d1) <= ratio on exact distances; the bound pre-filters,
    // which may only defer, use a slightly inflated ratio^2 so that rounding in the division / sqrt can never reject a match
    P.test_mode = test_mode;
    P.ratio = ratio;
    P.ratio_sq = (test_mode == 0) ? ratio * ratio : ratio * ratio * (1.0 + 1e-9);
    // whether d0 == d1 > 0 passes the final test (the kernels' ratio_pass): at ratio 1.0 in test mode 1, as in the symmetric
    // pass of bundler --add_images, the choice among keys tied for the nearest distance becomes part of the output
    P.ties_pass = (test_mode == 0) ? (ratio * ratio > 1.0) : (ratio >= 1.0);
    P.neg2 = -2;
    P.cand = (int32_t *) (S + o_cand); P.cand_cap = (int32_t) cap;
    P.hard = (int32_t *) (S + o_hard);
    // 1 = bound epilogue (default; needs every image to fit the kernel's norm staging buffer), 0 = exact chunk minima
    int32_t max_img_rows = 0;
    for (int i = 0; i < db->N; i++) max_img_rows = std::max(max_img_rows, db->img_rows[(size_t) i]);
    P.epi_mode = (env_int("BSFM_MATCH_EPILOGUE", 1) == 1 && max_img_rows <= TC_NORM_CAP) ? 1 : 0;
    // CTA-pair kernel (clusters of two sharing every database tile through TMA multicast: half the L2 -> SM traffic) and the
    // four-part variant (four N = 64 register accumulators per tile instead of two N = 128); both bound epilogue only
    const bool pair_mode = env_int("BSFM_MATCH_PAIR", 0) != 0;
    const bool quad_mode = env_int("BSFM_MATCH_QUAD", 0) != 0;
    P.match_slot = (uint32_t *) (S + o_slot_a); P.match_idx2 = (int32_t *) (S + o_idx_a); P.match_cap = (int32_t) cap;
    P.counters = (int32_t *) (S + o_cnt);

    // the dynamic shared-memory limit is a per-device (per-context) function attribute: set it once per device
    static std::atomic<int> attr_done[64];
    if (db->device < 0 || db->device >= 64 || !attr_done[db->device].load(std::memory_order_acquire)) {
        BSFM_CUDA_TRY(cudaFuncSetAttribute(match_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_ALLOC));
        BSFM_CUDA_TRY(cudaFuncSetAttribute(match_tc_bound_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_ALLOC));
        BSFM_CUDA_TRY(cudaFuncSetAttribute(match_tc_quad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_ALLOC));
        BSFM_CUDA_TRY(cudaFuncSetAttribute(match_tc_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_ALLOC));
        if (db->device >= 0 && db->device < 64) attr_done[db->device].store(1, std::memory_order_release);
    }

    float ms_search = 0.f;
    // launches cover whole database images: the sort keys of an image's queries span all of its tiles
    size_t run_pos = 0;
    for (int64_t u0 = 0; u0 < nunits;) {
        int64_t u1 = u0;
        while (run_pos < run.size() && (u1 == u0 || (int64_t) run[run_pos].unit0 + run[run_pos].nunits - u0 <= chunk_units)) {
            u1 = (int64_t) run[run_pos].unit0 + run[run_pos].nunits;
            run_pos++;
        }
        P.unit_begin = (int32_t) u0; P.unit_end = (int32_t) u1;
        BSFM_CUDA_TRY(cudaMemsetAsync(P.counters, 0, 64, db->stream));
        BSFM_CUDA_TRY(cudaEventRecord(db->ev[1], db->stream));
        int32_t h_cnt[4] = {0, 0, 0, 0};
        if (kernel_sel == BSFM_MATCH_KERNEL_DP4A) {
            match_dp4a_kernel<<<(unsigned) (u1 - u0), 256, 0, db->stream>>>(P);
            BSFM_KERNEL_CHECK();
            BSFM_CUDA_TRY(cudaEventRecord(db->ev[2], db->stream));
        } else {
            const int grid = (int) std::min<int64_t>(db->num_sms, u1 - u0);
            if (P.epi_mode == 1 && pair_mode && (u1 - u0) % 2 == 0) {
                cudaLaunchConfig_t cfg = {};
                cfg.gridDim = dim3((unsigned) (2 * std::min<int64_t>(std::max(1, db->num_sms / 2), (u1 - u0) / 2)));
                cfg.blockDim = dim3(TC_THREADS);
                cfg.dynamicSmemBytes = TC_SMEM_ALLOC;
                cfg.stream = db->stream;
                cudaLaunchAttribute attr[1];
                attr[0].id = cudaLaunchAttributeClusterDimension;
                attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
                cfg.attrs = attr; cfg.numAttrs = 1;
                BSFM_CUDA_TRY(cudaLaunchKernelEx(&cfg, match_tc_pair_kernel, P));
            } else if (P.epi_mode == 1 && quad_mode) match_tc_quad_kernel<<<grid, TC_THREADS, TC_SMEM_ALLOC, db->stream>>>(P);
            else if (P.epi_mode == 1) match_tc_bound_kernel<<<grid, TC_THREADS, TC_SMEM_ALLOC, db->stream>>>(P);
            else match_tc_kernel<<<grid, TC_THREADS, TC_SMEM_ALLOC, db->stream>>>(P);
            BSFM_KERNEL_CHECK();
            BSFM_CUDA_TRY(cudaEventRecord(db->ev[2], db->stream));
            BSFM_CUDA_TRY(cudaMemcpyAsync(h_cnt, P.counters, sizeof h_cnt, cudaMemcpyDeviceToHost, db->stream));
            BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
            if (h_cnt[2]) { set_error("bsfm_match_run: candidate buffer overflow (internal)"); return BSFM_ERR_CUDA; }
            const int ncand = h_cnt[0];
            if (ncand > 0) {
                const int64_t threads = (int64_t) ncand * 32;
                match_verify_kernel<<<(unsigned) ((threads + 255) / 256), 256, 0, db->stream>>>(P, ncand);
                BSFM_KERNEL_CHECK();
                BSFM_CUDA_TRY(cudaMemcpyAsync(h_cnt, P.counters, sizeof h_cnt, cudaMemcpyDeviceToHost, db->stream));
                BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
                if (h_cnt[2]) { set_error("bsfm_match_run: hard-row buffer overflow (internal)"); return BSFM_ERR_CUDA; }
                const int nhard = h_cnt[3];
                db->hard_rows += nhard; db->cand_rows += ncand;
                if (nhard > 0) {
                    match_fullscan_kernel<<<(unsigned) nhard, 256, 0, db->stream>>>(P, nhard);
                    BSFM_KERNEL_CHECK();
                }
            }
        }
        BSFM_CUDA_TRY(cudaMemcpyAsync(h_cnt, P.counters, sizeof h_cnt, cudaMemcpyDeviceToHost, db->stream));
        BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
        {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, db->ev[1], db->ev[2]);
            ms_search += ms;
        }
        if (h_cnt[2]) { set_error("bsfm_match_run: match buffer overflow (internal)"); return BSFM_ERR_CUDA; }
        const int nmatch = h_cnt[1];
        if (nmatch > 0) {
            rc = grow_matches(db, db->total_matches + nmatch);
            if (rc != BSFM_OK) { return rc; }
            size_t tb = cub_bytes;
            int end_bit = 1;
            while (end_bit < 32 && ((uint64_t) 1 << end_bit) < (uint64_t) (u1 - u0) * TILE_Q) end_bit++;
            cub::DeviceRadixSort::SortPairs(S + o_cub, tb, (const uint32_t *) (S + o_slot_a), (uint32_t *) (S + o_slot_b),
                                            (const int32_t *) (S + o_idx_a), (int32_t *) (S + o_idx_b), nmatch, 0, end_bit, db->stream);
            count_launch(3);
            BSFM_CUDA_TRY(cudaGetLastError());
            match_finalize_kernel<<<(nmatch + 255) / 256, 256, 0, db->stream>>>((const uint32_t *) (S + o_slot_b), (const int32_t *) (S + o_idx_b),
                                                                                nmatch, d_run, K, (int) u0, db->d_tile_img, db->d_img_doff, db->d_perm,
                                                                                db->d_matches + 2 * db->total_matches, db->d_pair_counts);
            BSFM_KERNEL_CHECK();
            db->total_matches += nmatch;
        }
        u0 = u1;
    }
    BSFM_CUDA_TRY(cudaEventRecord(db->ev[3], db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    float ms_total = 0.f;
    cudaEventElapsedTime(&ms_total, db->ev[0], db->ev[3]);
    db->ms[0] = ms_search; db->ms[1] = ms_total - ms_search; db->ms[2] = ms_total;
    db->launches = (int) (g_kernel_launches.load() - launches0);
    if (env_int("BSFM_MATCH_VERBOSE", 0))
        fprintf(stderr, "[bsfm_match_run] candidates %lld, hard rows %lld, matches %lld\n", (long long) db->cand_rows,
                (long long) db->hard_rows, (long long) db->total_matches);
    return db->total_matches;
}

extern "C" {

bsfm_keydb *bsfm_keydb_create(const uint8_t *keys, const int64_t *key_off, int num_images)
{
    clear_error();
    bsfm_keydb *db = new bsfm_keydb();
    if (keydb_build(db, keys, false, key_off, num_images) != BSFM_OK) { bsfm_keydb_destroy(db); return nullptr; }
    return db;
}

bsfm_keydb *bsfm_keydb_create_dev(const uint8_t *keys_dev, const int64_t *key_off, int num_images)
{
    clear_error();
    bsfm_keydb *db = new bsfm_keydb();
    if (keydb_build(db, keys_dev, true, key_off, num_images) != BSFM_OK) { bsfm_keydb_destroy(db); return nullptr; }
    return db;
}

void bsfm_keydb_destroy(bsfm_keydb *db)
{
    if (!db) return;
    cudaFree(db->d_keys_sw); cudaFree(db->d_norms); cudaFree(db->d_perm); cudaFree(db->d_tile_img); cudaFree(db->d_img_doff);
    cudaFree(db->d_pair_counts); cudaFree(db->d_matches); cudaFree(db->scratch); cudaFree(db->d_gather_counts); cudaFree(db->d_gather_matches);
    for (int e = 0; e < 4; e++) if (db->ev[e]) cudaEventDestroy(db->ev[e]);
    if (db->stream) cudaStreamDestroy(db->stream);
    delete db;
}

int64_t bsfm_match_num_pairs(int num_images, int window_radius)
{
    int64_t p = 0;
    for (int i = 0; i < num_images; i++) p += i - start_image(i, window_radius);
    return p;
}

int64_t bsfm_match_run(bsfm_keydb *db, int img_begin, int img_end, int window_radius, double ratio)
{
    return match_run_impl(db, img_begin, img_end, window_radius, ratio);
}

int64_t bsfm_match_shard_pairs(bsfm_keydb *db) { return db ? db->shard_pairs : BSFM_ERR_ARG; }

int bsfm_match_fetch(bsfm_keydb *db, int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap)
{
    clear_error();
    if (!db) { set_error("bsfm_match_fetch: null db"); return BSFM_ERR_ARG; }
    if (pair_cap < db->shard_pairs || match_cap < db->total_matches) {
        set_error("bsfm_match_fetch: need %lld pairs / %lld matches, got %lld / %lld", (long long) db->shard_pairs,
                  (long long) db->total_matches, (long long) pair_cap, (long long) match_cap);
        return BSFM_ERR_CAPACITY;
    }
    if (db->shard_pairs > 0)
        BSFM_CUDA_TRY(cudaMemcpyAsync(pair_counts, db->d_pair_counts, (size_t) db->shard_pairs * sizeof(int32_t), cudaMemcpyDeviceToHost, db->stream));
    if (db->total_matches > 0)
        BSFM_CUDA_TRY(cudaMemcpyAsync(matches, db->d_matches, (size_t) db->total_matches * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    return BSFM_OK;
}

int bsfm_match_result_dev(bsfm_keydb *db, const int32_t **pair_counts_dev, int64_t *num_pairs,
                          const int32_t **matches_dev, int64_t *num_matches)
{
    if (!db) { set_error("bsfm_match_result_dev: null db"); return BSFM_ERR_ARG; }
    if (pair_counts_dev) *pair_counts_dev = db->d_pair_counts;
    if (num_pairs) *num_pairs = db->shard_pairs;
    if (matches_dev) *matches_dev = db->d_matches;
    if (num_matches) *num_matches = db->total_matches;
    return BSFM_OK;
}

int bsfm_match_copy_result_dev(bsfm_keydb *db, int32_t *pair_counts_dst_dev, int32_t *matches_dst_dev)
{
    clear_error();
    if (!db) { set_error("bsfm_match_copy_result_dev: null db"); return BSFM_ERR_ARG; }
    if (db->shard_pairs > 0 && pair_counts_dst_dev)
        BSFM_CUDA_TRY(cudaMemcpyAsync(pair_counts_dst_dev, db->d_pair_counts, (size_t) db->shard_pairs * sizeof(int32_t), cudaMemcpyDeviceToDevice, db->stream));
    if (db->total_matches > 0 && matches_dst_dev)
        BSFM_CUDA_TRY(cudaMemcpyAsync(matches_dst_dev, db->d_matches, (size_t) db->total_matches * 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    return BSFM_OK;
}

int bsfm_match_last_timing(bsfm_keydb *db, float ms[3], int *launches)
{
    if (!db) { set_error("bsfm_match_last_timing: null db"); return BSFM_ERR_ARG; }
    if (ms) { ms[0] = db->ms[0]; ms[1] = db->ms[1]; ms[2] = db->ms[2]; }
    if (launches) *launches = db->launches;
    return BSFM_OK;
}

int64_t bsfm_match_all_pairs(const uint8_t *keys, const int64_t *key_off, int num_images, int window_radius, double ratio,
                             int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap)
{
    bsfm_keydb *db = bsfm_keydb_create(keys, key_off, num_images);
    if (!db) return BSFM_ERR_CUDA;
    int64_t total = bsfm_match_run(db, 0, num_images, window_radius, ratio);
    if (total >= 0) {
        int rc = bsfm_match_fetch(db, pair_counts, pair_cap, matches, match_cap);
        if (rc != BSFM_OK) total = rc;
    }
    bsfm_keydb_destroy(db);
    return total;
}

}  // extern "C"

/* MatchKeys(k1 = queries, k2 = database): image 0 = k1, image 1 = k2, the single pair (0,1).
 *
 * The unmodified KeyMatchFull main calls this once per image pair with the SAME host buffers over and over
 * (src/KeyMatchFull.cpp:105-151: keys live for the whole run, SURVEY.md 8b).  Prepared device images (norm-sorted,
 * swizzled) are therefore cached per (host pointer, key count, 64-bit content hash): a repeated image costs one hash of
 * its 640 KB instead of an upload, ~10 cudaMallocs and a segmented sort, and the pair runs on a persistent two-image
 * database filled by device-to-device copies. */
namespace {
struct CachedImage { const uint8_t *host; int n; uint64_t hash; bsfm_keydb *db; uint64_t last_use; size_t bytes; };
struct PairCache {
    std::mutex mu;
    std::vector<CachedImage> imgs;
    uint64_t tick = 0;
    size_t bytes = 0;
    int device = -1;
    bsfm_keydb *pair = nullptr;
    int64_t pair_rows_cap = 0;
    void flush()
    {
        for (auto &c : imgs) bsfm_keydb_destroy(c.db);
        imgs.clear(); bytes = 0;
        if (pair) bsfm_keydb_destroy(pair);
        pair = nullptr; pair_rows_cap = 0;
    }
};
PairCache g_pair_cache;

uint64_t hash_keys(const uint8_t *p, size_t bytes)      // bytes is a multiple of 128
{
    uint64_t h[8] = {0x9E3779B97F4A7C15ull, 0xC2B2AE3D27D4EB4Full, 0x165667B19E3779F9ull, 0x27D4EB2F165667C5ull,
                     0x85EBCA77C2B2AE63ull, 0xFF51AFD7ED558CCDull, 0xC4CEB9FE1A85EC53ull, 0x2545F4914F6CDD1Dull};
    const size_t nw = bytes / 8;
    for (size_t w = 0; w + 8 <= nw; w += 8) {
        uint64_t v[8];
        memcpy(v, p + w * 8, 64);
        for (int q = 0; q < 8; q++) { h[q] = (h[q] ^ v[q]) * 0x100000001B3ull; h[q] ^= h[q] >> 29; }
    }
    uint64_t r = bytes;
    for (int q = 0; q < 8; q++) r = (r ^ h[q]) * 0x9FB21C651E98DF25ull;
    return r ^ (r >> 32);
}

// cached one-image database of (k, n); builds it on a miss.  Caller holds the mutex.
bsfm_keydb *cached_image(PairCache &C, const uint8_t *k, int n)
{
    const uint64_t h = hash_keys(k, (size_t) n * DESC_BYTES);
    for (auto &c : C.imgs)
        if (c.n == n && c.hash == h) { c.last_use = ++C.tick; c.host = k; return c.db; }
    const size_t limit_bytes = (size_t) 8 << 30;
    while (!C.imgs.empty() && (C.imgs.size() >= 8192 || C.bytes > limit_bytes)) {      // evict the least recently used image
        size_t victim = 0;
        for (size_t q = 1; q < C.imgs.size(); q++) if (C.imgs[q].last_use < C.imgs[victim].last_use) victim = q;
        C.bytes -= C.imgs[victim].bytes;
        bsfm_keydb_destroy(C.imgs[victim].db);
        C.imgs.erase(C.imgs.begin() + (long) victim);
    }
    int64_t off[2] = {0, n};
    bsfm_keydb *db = new bsfm_keydb();
    if (keydb_build(db, k, false, off, 1) != BSFM_OK) { bsfm_keydb_destroy(db); return nullptr; }
    CachedImage c{k, n, h, db, ++C.tick, (size_t) db->drows * (DESC_BYTES + 8)};
    C.bytes += c.bytes;
    C.imgs.push_back(c);
    return db;
}

// the persistent two-image database, (re)allocated for at least `rows` device rows
int ensure_pair_db(PairCache &C, int64_t rows, int device)
{
    if (C.pair && C.pair_rows_cap >= rows) return BSFM_OK;
    if (C.pair) bsfm_keydb_destroy(C.pair);
    C.pair = nullptr; C.pair_rows_cap = 0;
    const int64_t cap = rows + rows / 4 + 4 * IMG_PAD;
    bsfm_keydb *db = new bsfm_keydb();
    db->N = 2; db->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete db; set_error("cudaGetDeviceProperties failed"); return BSFM_ERR_CUDA; }
    db->num_sms = prop.multiProcessorCount;
    C.pair = db;      // bsfm_keydb_destroy releases whatever was allocated if a step below fails
    BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&db->stream, cudaStreamNonBlocking));
    for (int e = 0; e < 4; e++) BSFM_CUDA_TRY(cudaEventCreate(&db->ev[e]));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_keys_sw, (size_t) cap * DESC_BYTES));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_norms, (size_t) cap * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_perm, (size_t) cap * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_tile_img, (size_t) (cap / TILE_Q) * sizeof(int32_t)));
    BSFM_CUDA_TRY(cudaMalloc(&db->d_img_doff, 3 * sizeof(int32_t)));
    C.pair_rows_cap = cap;
    return BSFM_OK;
}

int match_pair_cached(const uint8_t *k1, int n1, const uint8_t *k2, int n2, double ratio, int test_mode, int32_t *out_pairs, int cap)
{
    PairCache &C = g_pair_cache;
    std::lock_guard<std::mutex> lock(C.mu);
    int dev = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    if (dev != C.device) { C.flush(); C.device = dev; }
    bsfm_keydb *a = cached_image(C, k1, n1);
    if (!a) return BSFM_ERR_CUDA;
    bsfm_keydb *b = cached_image(C, k2, n2);      // may evict, never the entry just touched (it is the most recent)
    if (!b) return BSFM_ERR_CUDA;
    const int32_t rows_a = a->img_rows[0], rows_b = b->img_rows[0];
    int rc = ensure_pair_db(C, (int64_t) rows_a + rows_b + IMG_PAD, dev);
    if (rc != BSFM_OK) return rc;
    bsfm_keydb *db = C.pair;
    db->key_off = {0, n1, (int64_t) n1 + n2};
    db->doff = {0, rows_a, rows_a + rows_b};
    db->img_rows = {rows_a, rows_b};
    db->drows = (int64_t) rows_a + rows_b + IMG_PAD;
    std::vector<int32_t> tile_img((size_t) (db->drows / TILE_Q), -1);
    for (int32_t t = 0; t < rows_a / TILE_Q; t++) tile_img[(size_t) t] = 0;
    for (int32_t t = rows_a / TILE_Q; t < (rows_a + rows_b) / TILE_Q; t++) tile_img[(size_t) t] = 1;
    cudaStream_t st = db->stream;
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_tile_img, tile_img.data(), tile_img.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_img_doff, db->doff.data(), 3 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    // image rows keep their swizzled layout under a copy to any row offset that is a multiple of 8 (here: of 256)
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_keys_sw, a->d_keys_sw, (size_t) rows_a * DESC_BYTES, cudaMemcpyDeviceToDevice, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_norms, a->d_norms, (size_t) rows_a * 4, cudaMemcpyDeviceToDevice, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_perm, a->d_perm, (size_t) rows_a * 4, cudaMemcpyDeviceToDevice, st));
    const size_t rb = (size_t) rows_b + IMG_PAD;      // with the spare padded tile that keeps 256-row reads in bounds
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_keys_sw + (size_t) rows_a * DESC_BYTES, b->d_keys_sw, rb * DESC_BYTES, cudaMemcpyDeviceToDevice, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_norms + rows_a, b->d_norms, rb * 4, cudaMemcpyDeviceToDevice, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(db->d_perm + rows_a, b->d_perm, rb * 4, cudaMemcpyDeviceToDevice, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));      // tile_img is a host temporary
    int64_t total = match_run_impl(db, 1, 2, -1, ratio, test_mode);
    if (total < 0) return (int) total;
    if (total > 0) {
        std::vector<int32_t> m((size_t) total * 2);
        int32_t pc = 0;
        rc = bsfm_match_fetch(db, &pc, 1, m.data(), total);
        if (rc != BSFM_OK) return rc;
        const int64_t ncopy = std::min<int64_t>(total, cap);
        if (ncopy > 0 && out_pairs) memcpy(out_pairs, m.data(), (size_t) ncopy * 2 * sizeof(int32_t));
    }
    return (int) std::min<int64_t>(total, INT_MAX);
}
}  // namespace

extern "C" {
int bsfm_match_pair(const uint8_t *k1, int n1, const uint8_t *k2, int n2, double ratio, int32_t *out_pairs, int cap)
{
    return bsfm_match_pair_test(k1, n1, k2, n2, ratio, BSFM_RATIO_TEST_KEYS2A, out_pairs, cap);
}

int bsfm_match_pair_test(const uint8_t *k1, int n1, const uint8_t *k2, int n2, double ratio, int ratio_test, int32_t *out_pairs, int cap)
{
    clear_error();
    if (n1 < 0 || n2 < 0 || cap < 0) { set_error("bsfm_match_pair: negative size"); return BSFM_ERR_ARG; }
    if (ratio_test != BSFM_RATIO_TEST_KEYS2A && ratio_test != BSFM_RATIO_TEST_KEYS) { set_error("bsfm_match_pair_test: unknown ratio test %d", ratio_test); return BSFM_ERR_ARG; }
    int rc = require_device();
    if (rc != BSFM_OK) return rc;
    if (n1 == 0 || n2 == 0) return 0;
    return match_pair_cached(k1, n1, k2, n2, ratio, ratio_test, out_pairs, cap);
}

/* ---- multi-GPU behind the C ABI (SURVEY.md 8e; KeyMatchFull.cpp:105-151 sharded by database image) --------------------- */
int bsfm_comm_unique_id(unsigned char id[BSFM_COMM_ID_BYTES])
{
    clear_error();
    NcclApi &nc = nccl_api();
    if (!nc.ok) { set_error("NCCL (libnccl.so.2) could not be loaded: the multi-GPU entry points need it"); return BSFM_ERR_UNSUPPORTED; }
    static_assert(sizeof(ncclUniqueId) <= BSFM_COMM_ID_BYTES, "id buffer");
    ncclUniqueId u;
    BSFM_NCCL_TRY(nc.GetUniqueId(&u));
    memset(id, 0, BSFM_COMM_ID_BYTES);
    memcpy(id, &u, sizeof u);
    return BSFM_OK;
}

bsfm_comm *bsfm_comm_create(const unsigned char id[BSFM_COMM_ID_BYTES], int rank, int world_size)
{
    clear_error();
    if (require_device() != BSFM_OK) return nullptr;
    NcclApi &nc = nccl_api();
    if (!nc.ok) { set_error("NCCL (libnccl.so.2) could not be loaded: the multi-GPU entry points need it"); return nullptr; }
    if (!id || world_size < 1 || rank < 0 || rank >= world_size) { set_error("bsfm_comm_create: bad arguments"); return nullptr; }
    bsfm_comm *c = new bsfm_comm();
    c->rank = rank; c->world = world_size;
    if (cudaGetDevice(&c->device) != cudaSuccess) { delete c; set_error("cudaGetDevice failed"); return nullptr; }
    ncclUniqueId u;
    memcpy(&u, id, sizeof u);
    ncclResult_t r = nc.CommInitRank(&c->comm, world_size, u, rank);
    if (r != ncclSuccess) { set_error("ncclCommInitRank failed: %s", nc.GetErrorString(r)); delete c; return nullptr; }
    // the first collectives of a communicator set up its channels and, for large messages, its bulk-protocol buffers (tens to
    // hundreds of ms): pay that here with one small and one 4 MB-per-rank all-gather, not inside the first real call
    if (world_size > 1) {
        const size_t per = (size_t) 1 << 20;
        int32_t *d = nullptr;
        if (cudaMalloc(&d, (size_t) world_size * per * sizeof(int32_t)) == cudaSuccess) {
            cudaMemset(d, 0, (size_t) world_size * per * sizeof(int32_t));
            nc.AllGather(d + rank, d, 1, ncclInt32, c->comm, (cudaStream_t) 0);
            nc.AllGather(d + rank * per, d, per, ncclInt32, c->comm, (cudaStream_t) 0);
            nc.Broadcast(d, d, 1024, ncclInt32, 0, c->comm, (cudaStream_t) 0);
            cudaStreamSynchronize((cudaStream_t) 0);
            cudaFree(d);
        }
    }
    return c;
}

void bsfm_comm_destroy(bsfm_comm *c)
{
    if (!c) return;
    if (c->comm) nccl_api().CommDestroy(c->comm);
    delete c;
}

bsfm_keydb *bsfm_keydb_create_sharded(bsfm_comm *comm, const uint8_t *keys, const int64_t *key_off, int num_images)
{
    clear_error();
    if (!comm) { set_error("bsfm_keydb_create_sharded: null communicator"); return nullptr; }
    bsfm_keydb *db = new bsfm_keydb();
    if (keydb_build(db, keys, false, key_off, num_images, comm) != BSFM_OK) { bsfm_keydb_destroy(db); return nullptr; }
    return db;
}

int bsfm_match_shard_range(const int64_t *key_off, int num_images, int window_radius, int world_size, int rank, int *img_begin, int *img_end)
{
    clear_error();
    if (!key_off || num_images < 0 || world_size < 1 || rank < 0 || rank >= world_size || !img_begin || !img_end) { set_error("bsfm_match_shard_range: bad arguments"); return BSFM_ERR_ARG; }
    // contiguous database-image ranges of (nearly) equal work n_i * sum_{j in window} n_j (the rule of keymatch.shard_images)
    std::vector<double> work((size_t) num_images);
    double total = 0.0;
    for (int i = 0; i < num_images; i++) {
        const int s0 = start_image(i, window_radius);
        work[(size_t) i] = (double) (key_off[i + 1] - key_off[i]) * (double) (key_off[i] - key_off[s0]);
        total += work[(size_t) i];
    }
    std::vector<int> bounds;
    bounds.push_back(0);
    double acc = 0.0;
    int r = 1;
    for (int i = 0; i < num_images; i++) {
        acc += work[(size_t) i];
        while (r < world_size && acc >= total * r / world_size) { bounds.push_back(i + 1); r++; }
    }
    while ((int) bounds.size() < world_size) bounds.push_back(num_images);
    bounds.push_back(num_images);
    for (size_t q = 1; q < bounds.size(); q++) bounds[q] = std::max(std::min(bounds[q], num_images), bounds[q - 1]);
    *img_begin = bounds[(size_t) rank]; *img_end = bounds[(size_t) rank + 1];
    return BSFM_OK;
}

int64_t bsfm_match_allgather(bsfm_comm *comm, bsfm_keydb *db)
{
    clear_error();
    if (!comm || !db) { set_error("bsfm_match_allgather: null argument"); return BSFM_ERR_ARG; }
    NcclApi &nc = nccl_api();
    const int W = comm->world;
    BSFM_CUDA_TRY(cudaSetDevice(db->device));
    // 1. sizes of every rank's table
    int64_t *d_sizes = nullptr;
    BSFM_CUDA_TRY(cudaMalloc(&d_sizes, (size_t) W * 2 * sizeof(int64_t)));
    struct Guard { void *q; ~Guard() { cudaFree(q); } } guard{d_sizes};
    const int64_t mine[2] = {db->shard_pairs, db->total_matches};
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_sizes + 2 * comm->rank, mine, sizeof mine, cudaMemcpyHostToDevice, db->stream));
    BSFM_NCCL_TRY(nc.AllGather(d_sizes + 2 * comm->rank, d_sizes, 2, ncclInt64, comm->comm, db->stream));
    std::vector<int64_t> sizes((size_t) W * 2);
    BSFM_CUDA_TRY(cudaMemcpyAsync(sizes.data(), d_sizes, sizes.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    int64_t tp = 0, tm = 0;
    for (int r = 0; r < W; r++) { tp += sizes[(size_t) 2 * r]; tm += sizes[(size_t) 2 * r + 1]; }
    if (tp > db->gather_pair_cap) {
        cudaFree(db->d_gather_counts); db->d_gather_counts = nullptr; db->gather_pair_cap = 0;
        BSFM_CUDA_TRY(cudaMalloc(&db->d_gather_counts, (size_t) std::max<int64_t>(tp, 1) * sizeof(int32_t)));
        db->gather_pair_cap = std::max<int64_t>(tp, 1);
    }
    if (tm > db->gather_match_cap) {
        cudaFree(db->d_gather_matches); db->d_gather_matches = nullptr; db->gather_match_cap = 0;
        BSFM_CUDA_TRY(cudaMalloc(&db->d_gather_matches, (size_t) std::max<int64_t>(tm, 1) * 2 * sizeof(int32_t)));
        db->gather_match_cap = std::max<int64_t>(tm, 1);
    }
    // 2. payload: rank r's counts and matches go to their offsets in the concatenated table (one grouped broadcast per rank:
    //    shards are contiguous database-image ranges in rank order, so the concatenation IS the KeyMatchFull order)
    BSFM_NCCL_TRY(nc.GroupStart());
    int64_t op = 0, om = 0;
    for (int r = 0; r < W; r++) {
        const int64_t np = sizes[(size_t) 2 * r], nm = sizes[(size_t) 2 * r + 1];
        if (np > 0) BSFM_NCCL_TRY(nc.Broadcast(db->d_pair_counts, db->d_gather_counts + op, (size_t) np, ncclInt32, r, comm->comm, db->stream));
        if (nm > 0) BSFM_NCCL_TRY(nc.Broadcast(db->d_matches, db->d_gather_matches + 2 * om, (size_t) nm * 2, ncclInt32, r, comm->comm, db->stream));
        op += np; om += nm;
    }
    BSFM_NCCL_TRY(nc.GroupEnd());
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    db->gather_pairs = tp; db->gather_matches = tm;
    return tm;
}

int bsfm_match_gathered_fetch(bsfm_keydb *db, int64_t *num_pairs, int64_t *num_matches, int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap)
{
    clear_error();
    if (!db) { set_error("bsfm_match_gathered_fetch: null db"); return BSFM_ERR_ARG; }
    if (num_pairs) *num_pairs = db->gather_pairs;
    if (num_matches) *num_matches = db->gather_matches;
    if (!pair_counts && !matches) return BSFM_OK;
    if (pair_cap < db->gather_pairs || match_cap < db->gather_matches) {
        set_error("bsfm_match_gathered_fetch: need %lld pairs / %lld matches, got %lld / %lld", (long long) db->gather_pairs,
                  (long long) db->gather_matches, (long long) pair_cap, (long long) match_cap);
        return BSFM_ERR_CAPACITY;
    }
    if (db->gather_pairs > 0 && pair_counts)
        BSFM_CUDA_TRY(cudaMemcpyAsync(pair_counts, db->d_gather_counts, (size_t) db->gather_pairs * sizeof(int32_t), cudaMemcpyDefault, db->stream));
    if (db->gather_matches > 0 && matches)
        BSFM_CUDA_TRY(cudaMemcpyAsync(matches, db->d_gather_matches, (size_t) db->gather_matches * 2 * sizeof(int32_t), cudaMemcpyDefault, db->stream));
    BSFM_CUDA_TRY(cudaStreamSynchronize(db->stream));
    return BSFM_OK;
}

}  // extern "C"

#include <thread>
namespace {
struct MultiShared {
    const uint8_t *keys; const int64_t *key_off; int N, window; double ratio; int ngpus; const int *devices;
    unsigned char id[BSFM_COMM_ID_BYTES];
    int32_t *pair_counts; int64_t pair_cap; int32_t *matches; int64_t match_cap;
    std::vector<int64_t> result; std::vector<std::string> errors; std::vector<float> search_ms;
};
void multi_worker(MultiShared *S, int rank)
{
    auto fail = [&](int64_t code) { S->result[(size_t) rank] = code; S->errors[(size_t) rank] = last_error(); };
    if (cudaSetDevice(S->devices ? S->devices[rank] : rank) != cudaSuccess) { set_error("cudaSetDevice(%d) failed", S->devices ? S->devices[rank] : rank); return fail(BSFM_ERR_CUDA); }
    bsfm_comm *comm = bsfm_comm_create(S->id, rank, S->ngpus);
    if (!comm) return fail(BSFM_ERR_CUDA);
    bsfm_keydb *db = bsfm_keydb_create_sharded(comm, S->keys, S->key_off, S->N);
    int64_t total = BSFM_ERR_CUDA;
    if (db) {
        int b = 0, e = 0;
        bsfm_match_shard_range(S->key_off, S->N, S->window, S->ngpus, rank, &b, &e);
        total = bsfm_match_run(db, b, e, S->window, S->ratio);
        S->search_ms[(size_t) rank] = db->ms[0];
        // every rank must enter the collective, also after a local failure: contribute an empty table then
        if (total < 0) { S->errors[(size_t) rank] = last_error(); db->shard_pairs = 0; db->total_matches = 0; }
        const int64_t g = bsfm_match_allgather(comm, db);
        if (total >= 0) total = g;
        if (total >= 0 && rank == 0) {
            int rc = bsfm_match_gathered_fetch(db, nullptr, nullptr, S->pair_counts, S->pair_cap, S->matches, S->match_cap);
            if (rc != BSFM_OK) total = rc;
        }
    }
    if (total < 0 && S->errors[(size_t) rank].empty()) S->errors[(size_t) rank] = last_error();
    S->result[(size_t) rank] = total;
    if (db) bsfm_keydb_destroy(db);
    bsfm_comm_destroy(comm);
}
}  // namespace

extern "C" {
int64_t bsfm_match_all_pairs_multi(const uint8_t *keys, const int64_t *key_off, int num_images, int window_radius, double ratio,
                                   int ngpus, const int *devices, int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap)
{
    clear_error();
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device available: libbsfm_b200 has no CPU fallback"); return BSFM_ERR_NO_DEVICE; }
    if (ngpus < 1 || ngpus > ndev) { set_error("bsfm_match_all_pairs_multi: ngpus = %d but %d device(s) are visible", ngpus, ndev); return BSFM_ERR_ARG; }
    if (ngpus == 1 && !devices) return bsfm_match_all_pairs(keys, key_off, num_images, window_radius, ratio, pair_counts, pair_cap, matches, match_cap);
    MultiShared S;
    S.keys = keys; S.key_off = key_off; S.N = num_images; S.window = window_radius; S.ratio = ratio; S.ngpus = ngpus; S.devices = devices;
    S.pair_counts = pair_counts; S.pair_cap = pair_cap; S.matches = matches; S.match_cap = match_cap;
    S.result.assign((size_t) ngpus, BSFM_ERR_CUDA); S.errors.assign((size_t) ngpus, std::string()); S.search_ms.assign((size_t) ngpus, 0.f);
    int saved = 0;
    cudaGetDevice(&saved);
    int rc = bsfm_comm_unique_id(S.id);
    if (rc != BSFM_OK) return rc;
    std::vector<std::thread> threads;
    for (int r = 0; r < ngpus; r++) threads.emplace_back(multi_worker, &S, r);     // one host thread per GPU
    for (auto &t : threads) t.join();
    cudaSetDevice(saved);
    for (int r = 0; r < ngpus; r++)
        if (S.result[(size_t) r] < 0) { set_error("bsfm_match_all_pairs_multi: rank %d: %s", r, S.errors[(size_t) r].c_str()); return S.result[(size_t) r]; }
    return S.result[0];
}

/* releases the device images bsfm_match_pair keeps between calls */
void bsfm_match_pair_cache_clear(void)
{
    std::lock_guard<std::mutex> lock(g_pair_cache.mu);
    g_pair_cache.flush();
}

}  // extern "C"
