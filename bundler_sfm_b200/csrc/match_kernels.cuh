// match_kernels.cuh -- sm_90a kernels of the MATCH hot path (SURVEY.md K9).
//
// Reference semantics (file:line under /root/reference):
//   for each query key q of image j and database image i (j < i):
//     d(q,p) = sum_k ((int)q_k - (int)p_k)^2        lib/ann_1.1_char/src/kd_pr_search.cpp:200-209
//     (d0, nn0), d1 = two smallest over p in image i lib/ann_1.1_char/src/pr_queue_k.h:102-117
//     emit (q, nn0) iff (double)d0 < ratio*ratio*(double)d1        src/keys2a.cpp:362
//
// HBM layout (DESIGN.md): inside every image the keys are stored in ascending order of their squared norm
// (perm[] maps a device row back to the caller's index); every image is padded to a multiple of 256 descriptor rows; a row is
// 128 bytes; rows are stored in the UMMA "K-major, SWIZZLE_128B" canonical shared-memory image
// (8-row x 128-byte atoms, 16-byte chunk c of row r stored at chunk c ^ (r & 7)) so that a tile
// of rows is ONE contiguous TMA bulk copy and lands in shared memory ready for wgmma.
// norms[row] = |p|^2 (int32) for real rows, NORM_PAD (2^30) for padding rows.
//
// d = |q|^2 + |p|^2 - 2 q.p is exact in int32 (max 128*255^2 = 8,323,200).  The tensor core
// produces q.p (u8 x u8 -> s32, wgmma.mma_async); ranking uses t = |p|^2 - 2 q.p.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace bsfm {
namespace match {

constexpr int DESC_BYTES = 128;
constexpr int TILE_Q = 128;          // query rows per work unit (two warpgroups of wgmma M = 64)
constexpr int TILE_DB = 256;         // database rows per tile (two wgmma N = 128 halves)
constexpr int IMG_PAD = 256;         // per-image row padding
constexpr int CHUNK = 32;            // database columns per exact-epilogue chunk
constexpr int32_t NORM_PAD = 1 << 30;
constexpr int32_t NORM_PAD_HALF = 1 << 29;

// tensor-core kernel configuration (shared by kernel and launcher)
constexpr int TC_MATH_THREADS = 256;               // two consumer warpgroups: 64 query rows each
constexpr int TC_THREADS = TC_MATH_THREADS + 32;   // + one TMA producer warp
constexpr int TC_B_STAGES = 4;
constexpr int TC_A_BYTES = TILE_Q * DESC_BYTES;    // 16384
constexpr int TC_B_BYTES = TILE_DB * DESC_BYTES;   // 32768
constexpr int TC_SMEM_A = 0;
constexpr int TC_SMEM_B = 2 * TC_A_BYTES;
constexpr int TC_NORM_CAP = 8192;                  // norms of a whole database image kept in smem
constexpr int BCHUNK = 64;                         // columns per bound-epilogue chunk: width the verify kernel recomputes
constexpr int TC_SMEM_NALL = TC_SMEM_B + TC_B_STAGES * TC_B_BYTES;
constexpr int TC_SMEM_BAR = TC_SMEM_NALL + TC_NORM_CAP * 4;
constexpr int TC_SMEM_BYTES = TC_SMEM_BAR + 256;
constexpr int TC_SMEM_ALLOC = TC_SMEM_BYTES + 1024;  // slack for manual 1024-byte alignment
static_assert(TC_SMEM_ALLOC <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// One database image of a run (shard): all query tiles [atile0, atile0 + ntiles_q) are matched
// against rows [db_row0, db_row0 + npad).
struct RunImage {
    int32_t img;        // database image index i
    int32_t n;          // real keys in image i (>0)
    int32_t db_row0;    // first device row of image i
    int32_t ntiles_db;  // npad_i / 256
    int32_t atile0;     // first 128-row query tile (device row / 128) = doff[start_i] / 128
    int32_t start_img;  // first query image j
    int32_t unit0;      // first work unit of this image inside the run
    int32_t nunits;     // number of query tiles
    int64_t pair0;      // index of pair (start_img, i) in the shard's pair list
};

struct MatchParams {
    const uint8_t *keys_sw;     // swizzled padded descriptors
    const int32_t *norms;       // per device row (ascending inside every image)
    const int32_t *perm;        // per device row: index of the key in the caller's order (-1 for padding)
    const int32_t *tile_img;    // image of every 128-row tile
    const int32_t *img_doff;    // first device row of every image
    const RunImage *run_imgs;   // K entries, unit0 ascending
    int32_t num_run_imgs;
    int32_t unit_begin;         // units [unit_begin, unit_end) are processed by this launch
    int32_t unit_end;
    double ratio_sq;            // ratio*ratio evaluated on the host in double (keys2a.cpp:362); test mode 1: inflated by 1e-9
                                // (only the conservative pre-filters of the tensor-core epilogue read it there)
    double ratio;               // the ratio itself (test mode 1)
    int32_t test_mode;          // 0: (double) d0 < ratio^2 (double) d1          MatchKeys of keys2a.cpp:362 / :412
                                // 1: sqrt((double) d0 / (double) d1) <= ratio   MatchKeys of keys.cpp:786 (bundler --add_images)
    int32_t ties_pass;          // 1 iff d0 == d1 > 0 passes the ratio test (test mode 0 with ratio^2 > 1, test mode 1 with ratio >= 1):
                                // only then is it observable which of several keys tied for the nearest distance is returned.
                                // The rule is the smallest caller index (perm[]) among them, on every kernel.
    int32_t neg2;               // the constant -2 as a runtime value (see the epilogue of match_tc_kernel)
    int32_t epi_mode;           // 1 = bound epilogue (max tree on norm-sorted chunks), 0 = exact chunk minima
    // candidate list (tensor-core kernel): SoA int32 [7][cand_cap]: slot, qrow, db0, col0, nvalid, f5, f6
    //   exact mode: f5 = upper bound on d1, f6 = INT_MIN;  bound mode: f5 = L2, f6 = Uo (t-space bounds of the other chunks)
    int32_t *cand;
    int32_t *hard;              // [2][cand_cap]: slot, qrow of rows the bounds could not decide
    int32_t cand_cap;
    // match list (unordered): slot keys + idx2 values
    uint32_t *match_slot;
    int32_t *match_idx2;
    int32_t match_cap;
    int32_t *counters;          // [0] = #candidates, [1] = #matches, [2] = overflow flag, [3] = #hard rows
};

// the ratio test on an exact (d0, d1) pair -- or on bounds of d1: both forms are monotone in d1, so a test that passes with a
// lower bound of d1 passes with d1 itself
__device__ __forceinline__ bool ratio_pass(const MatchParams &P, int d0, int d1)
{
    if (P.test_mode == 0) return (double) d0 < P.ratio_sq * (double) d1;
    return sqrt((double) d0 / (double) d1) <= P.ratio;       // 0 / 0 = NaN: no match, as in the reference
}

// byte offset of 16-byte chunk c (0..7) of device row r in the swizzled layout
__host__ __device__ __forceinline__ size_t sw_chunk_offset(int64_t row, int c)
{
    return (size_t) (row >> 3) * 1024 + (size_t) (row & 7) * 128 + (size_t) ((c ^ (int) (row & 7)) << 4);
}

// Sort key of a match: queries of image j occupy the slot range that starts at the first tile of j for this
// database image; the key is that base plus the query's index in the CALLER's order, so sorting by key restores
// KeyMatchFull's order (i ascending, j ascending, query ascending) although rows are stored norm-sorted.
__device__ __forceinline__ uint32_t match_sort_key(const MatchParams &P, const RunImage &R, int64_t qrow)
{
    const int atile = (int) (qrow >> 7);
    const int j = P.tile_img[atile];
    const int base_unit = R.unit0 + (P.img_doff[j] >> 7) - R.atile0;
    return (uint32_t) (base_unit - P.unit_begin) * TILE_Q + (uint32_t) P.perm[qrow];
}

// find the run image that owns work unit u (binary search over unit0)
__device__ __forceinline__ int find_run_image(const RunImage *imgs, int K, int u)
{
    int lo = 0, hi = K - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (imgs[mid].unit0 <= u) lo = mid; else hi = mid - 1;
    }
    return lo;
}

}  // namespace match
}  // namespace bsfm
