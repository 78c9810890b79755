// ba_chol_large.cuh -- shared definitions of the large-system Cholesky path (ba_chol_large.cu) and the dataflow kernel.
#pragma once
#include <algorithm>
#include <cuda_runtime.h>
#include <cstdint>
#include <cmath>

namespace bsfm {
namespace ba {

struct Scalars;

constexpr int LNB = 32;          // sub-block
constexpr int LNBO = 256;        // outer panel
constexpr int CHOL_LARGE_MIN = 1536;     // systems above this size are throughput-bound: 256-column panel path
// geometry of the large path's zero-block skip (ba_chol_large.cu), shared with the camera order that feeds it (ba_order.cu):
// the panel solve flags 64-row slabs, the trailing update keeps 128 x 128 tiles from a list of at most 128 row blocks, and the
// dataflow kernel takes over once at most CHOL_TAIL_MAX columns remain (BSFM_BA_CHOL_TAIL)
constexpr int CHOL_SLAB = 64, CHOL_TILE = 128, CHOL_MAX_RB = 128, CHOL_TAIL_MAX = 640;
int chol_solve_large(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *xinv_ws, double *x, Scalars *sc);
// doubles of linear-solver workspace behind the 32 x 32 inverses: back-substitution scratch (small path) or the 256 x 256 panel inverses (large path)
constexpr int DF_MAX_N = 24 * LNB;       // largest system the dataflow path (ba_chol_dataflow.cu) takes: it needs (n + 1) x n doubles more
constexpr int DF_MAX_NBK = 20;           // and at most this many 32-column blocks (n <= 640)
// the large path's zero flags: one int per 64-row slab of every panel solve (rows below the panel + the right-hand side row),
// a stride of (n + 1) / 64 rounded up per panel
inline size_t chol_large_flag_count(int n) { return (size_t) ((n + LNBO - 1) / LNBO) * (size_t) ((n + 64) / 64); }
inline size_t chol_extra_ws_doubles(int n)
{
    // small systems: (n + 1) x n behind the scratch; large ones finish their last panels with the dataflow kernel: room for its
    // largest case, then the zero flags
    return (size_t) ((n + LNBO - 1) / LNBO) * LNBO * LNBO + (size_t) n + 64 + (size_t) (std::min(n, DF_MAX_N) + 1) * std::min(n, DF_MAX_N) + 64 +
           (chol_large_flag_count(n) + 1) / 2;
}
// doubles of the whole linv_ws workspace chol_solve takes for an n x n system: the 32 x 32 inverses, then the above
inline size_t chol_ws_doubles(int n) { return (size_t) ((n + LNB - 1) / LNB) * LNB * LNB + chol_extra_ws_doubles(n); }
// symmetric A (both triangles) + right-hand side in row n, factor out of place in Lmat, solution in x (ba_chol.cu)
int chol_solve(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *x, Scalars *sc);
// where the large path keeps that scratch inside linv_ws
inline size_t chol_large_pub_offset(int n) { return (size_t) ((n + LNB - 1) / LNB) * LNB * LNB + (size_t) ((n + LNBO - 1) / LNBO) * LNBO * LNBO + (size_t) n + 64; }
// and the zero flags behind it
inline size_t chol_large_flags_offset(int n) { return chol_large_pub_offset(n) + (size_t) (std::min(n, DF_MAX_N) + 1) * std::min(n, DF_MAX_N) + 64; }
int chol_dataflow_factor(cudaStream_t st, const double *A, double *Lmat, int ld, int n, double *linv_blocks, double *pub, Scalars *sc, bool *used);

}  // namespace ba
}  // namespace bsfm
