// ba_chol_large.cuh -- shared definitions of the large-system Cholesky path (ba_chol_large.cu) and the dataflow kernel.
#pragma once
#include <algorithm>
#include <cuda_runtime.h>
#include <cstdint>
#include <cmath>
#include <vector>

namespace bsfm {
namespace ba {

struct Scalars;
struct CholBand;

constexpr int LNB = 32;          // sub-block
constexpr int LNBO = 256;        // outer panel
constexpr int CHOL_LARGE_MIN = 1536;     // systems above this size are throughput-bound: 256-column panel path
// geometry of the large path's zero-block skip (ba_chol_large.cu), shared with the camera order that feeds it (ba_order.cu):
// the panel solve flags 64-row slabs, the trailing update keeps 128 x 128 tiles from a list of at most 128 row blocks, and the
// dataflow kernel takes over once at most CHOL_TAIL_MAX columns remain (BSFM_BA_CHOL_TAIL)
constexpr int CHOL_SLAB = 64, CHOL_TILE = 128, CHOL_MAX_RB = 128, CHOL_TAIL_MAX = 640;
int chol_solve_large(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *xinv_ws, double *x, Scalars *sc,
                     const CholBand *band = nullptr);
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
// Band plan of a large system whose rows have a narrow envelope (ba_order.cu: chol_band_plan; DESIGN.md 3.4 "Band
// factorisation").  Row i's first nonzero column first[i] is also that of L (Cholesky fill stays inside the row envelope), so
// in 32 x 32 tiles the factor lives in the tiles (rb, cb), env[rb] <= cb <= rb, plus the right-hand-side row nbk (env = 0).
// Tile (rb, cb) takes the rank-32 updates of steps max(env[rb], env[cb]) .. klast (cb - 1; cb - 2 for a diagonal tile, whose
// last update is the diagonal chain's look-ahead); the tiles with at least one such step are held by the worker CTAs of
// chol_band_kernel (ba_chol_dataflow.cu), two register slots each, assigned by interval colouring in order of first step.
constexpr int CHOL_BAND_MAX_N = 24 * 1024;      // the band back substitution keeps y (n doubles) in shared memory
// Mid-size systems (1537 .. 4096 unknowns: at most 13 panels ahead of the dataflow tail) keep the panel path whatever their
// envelope: it is the path the camera order is scored for (ba_order.cu: kept_tiles), and the band path's gain is measured on
// larger systems (config 3) only
constexpr int CHOL_BAND_MIN_N = 4096;
struct CholBandPlan {
    int n = 0, nbk = 0;
    int ntile = 0;            // tiles of the envelope, right-hand-side row included (the packed publish buffer)
    int max_live = 0;         // largest number of tiles that take updates at one step
    int workers = 0;          // worker CTAs the schedule uses
    bool fits = false;        // the schedule needs at most two slots per worker and the buffer fits the solver's workspace
    std::vector<int> env;     // nbk + 1
    std::vector<int> toff;    // nbk + 2: packed index of tile (rb, env[rb]); toff[nbk + 1] = ntile
    std::vector<int> sptr;    // 2 workers + 1: slot s of worker w holds sched[sptr[2 w + s] .. sptr[2 w + s + 1])
    std::vector<int> sched;   // rb << 16 | cb, each slot's tiles in increasing step
};
// first_col[i]: first nonzero column of row i (<= i); max_workers: worker CTAs available (SMs - 1)
void chol_band_plan(int n, const int *first_col, int max_workers, CholBandPlan &plan);
// the plan on the device (uploaded once per solve); env == nullptr: no plan, the panel path runs
struct CholBand {
    const int *env = nullptr, *toff = nullptr, *sptr = nullptr, *sched = nullptr;
    int ntile = 0, workers = 0;
};
// symmetric A (both triangles) + right-hand side in row n, factor out of place in Lmat, solution in x (ba_chol.cu).  band: the
// system's envelope plan (entries of A outside it are taken as zero), or null
int chol_solve(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *x, Scalars *sc, const CholBand *band = nullptr);
// where the large path keeps that scratch inside linv_ws
inline size_t chol_large_pub_offset(int n) { return (size_t) ((n + LNB - 1) / LNB) * LNB * LNB + (size_t) ((n + LNBO - 1) / LNBO) * LNBO * LNBO + (size_t) n + 64; }
// and the zero flags behind it
inline size_t chol_large_flags_offset(int n) { return chol_large_pub_offset(n) + (size_t) (std::min(n, DF_MAX_N) + 1) * std::min(n, DF_MAX_N) + 64; }
int chol_dataflow_factor(cudaStream_t st, const double *A, double *Lmat, int ld, int n, double *linv_blocks, double *pub, Scalars *sc, bool *used);
// the band path (ba_chol_dataflow.cu): one cooperative factorisation launch, its tiles published into the packed buffer `pub`
// (ntile x 1024 doubles) right behind the 32 x 32 inverses; then the envelope-bounded back substitution
inline size_t chol_band_capacity_tiles(int n) { return (size_t) ((n + LNBO - 1) / LNBO) * LNBO * LNBO / (LNB * LNB); }
int chol_band_factor(cudaStream_t st, const double *A, double *Lmat, int n, double *linv_ws, const CholBand &B, Scalars *sc);
int chol_band_backsolve(cudaStream_t st, const double *Lmat, int n, const double *linv_ws, const CholBand &B, double *x);

}  // namespace ba
}  // namespace bsfm
