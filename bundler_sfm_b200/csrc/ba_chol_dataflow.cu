// ba_chol_dataflow.cu -- dense SPD factorisation of SMALL reduced camera systems (n <= 640; config 2: 50 cameras -> 450) as ONE
// co-resident launch per factorisation; also finishes the last panels of large systems in place (ba_chol_large.cu), and factors
// large systems with a narrow row envelope whole (chol_band_kernel, below).
// Reference: dpotrf inside sba_Axb_Chol, lib/sba-1.5/sba_lapack.c:429.
//
// Small systems are bound by the chain of n sequential pivots and by L2 round trips, not by FLOPs.  The
// fused-step path (ba_chol.cu) pays one launch per 32 columns and a 16-warp, barrier-per-pivot factorisation of the diagonal tile in
// every CTA.  Here the whole factorisation is a dataflow over 32 x 32 tiles inside one cooperative launch, no grid-wide barrier:
//   CTA 0        owns the critical path.  Per 32-column step k: warp 0 factors the diagonal tile (warp_potf2_32_tc, ba_chol_potf2.cuh),
//                warp 1 assembles Z_kk = L_kk^-1 one panel behind it, warps 4..7 send Z_kk out the moment it exists, warps 2..3
//                fetch the look-ahead inputs as they arrive; then X <- X Z^T for the sub-diagonal block and the rank-32 update
//                of the NEXT diagonal tile, which never leaves shared memory.
//   CTAs 1..G-1  own the other tiles statically (at most two each) and keep them in REGISTERS (DMMA accumulator layout) through
//                all their rank-32 updates; a tile goes to global memory exactly once, when it is finished.  Per step: fetch the
//                two finished panel blocks of every owned tile, then Z_kk, X <- X Z^T strips and the update on the fp64 tensor cores.
//   transport    every 8-byte word that travels between CTAs is its own ready flag: it is written once into memory pre-filled
//                with an all-ones pattern and re-read by the consumer until it differs (no flag round trip, no fence).
// Same data contract as chol_solve (factor OUT OF PLACE in Lmat, right-hand side as matrix row n, inverses of the diagonal tiles in
// linv).  Waits are bounded: a word that never arrives sets sc->chol_fail = 2 instead of hanging the device.
// Design notes: DESIGN.md 3.4.
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"
#include "ba_chol_potf2.cuh"
#include "common.h"
#include <algorithm>
#include <atomic>
#include <cstdlib>

namespace bsfm {
namespace ba {

constexpr int DF_THREADS = 256;
constexpr long long DF_SPIN_LIMIT = 400000;      // polls of one L2 round trip each: a lost flag costs well under a second, never a hang
// The band kernel's workers may start their first tile hundreds of steps into the factorisation and wait for all of them:
// its bound grows with the step count (a step takes ~11 us; this allows well over a millisecond of polls per step)
constexpr long long DF_SPIN_PER_STEP = 4000;

// ---- data that is its own "ready" flag ----
// Everything that travels between CTAs (Z_kk blocks, finished tiles) is written exactly once per solve into memory the host
// pre-filled with an all-ones pattern (a NaN no arithmetic produces).  A consumer simply re-reads each 8-byte word until it is not
// the pattern: naturally aligned 8-byte accesses are single-copy atomic, so a word is either "not yet" or final.  Compared with a
// separate flag this removes one L2 round trip and the fence on each side of every hop (store, fence, flag | poll, load).
__device__ __forceinline__ double ld_strong(const double *p)
{
    double v;
    asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_strong(double *p, double v)
{
    asm volatile("st.relaxed.gpu.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ bool df_pending(double v) { return __double_as_longlong(v) == -1LL; }

// Fetch NE elements per thread: element i of this thread comes from src(i) (nullptr: not part of the tile, takes fill(i)) and is
// handed to put(i, value).  Re-reads the words that are still pending (bounded).
template <int NE, class Src, class Put>
__device__ __forceinline__ void df_fetch(Src src, Put put, Scalars *sc, long long spin_limit = DF_SPIN_LIMIT)
{
    double v[NE];
    unsigned pend = 0;
#pragma unroll
    for (int i = 0; i < NE; i++) {
        const double *p = src(i);
        v[i] = p ? ld_strong(p) : 0.0;
        if (p && df_pending(v[i])) pend |= 1u << i;
    }
    long long spins = 0;
    while (pend) {
#pragma unroll
        for (int i = 0; i < NE; i++) {
            if (pend & (1u << i)) {
                v[i] = ld_strong(src(i));
                if (!df_pending(v[i])) pend &= ~(1u << i);
            }
        }
        if (++spins > spin_limit) { sc->chol_fail = 2; break; }
        if (pend) __nanosleep(32);
    }
#pragma unroll
    for (int i = 0; i < NE; i++) put(i, v[i]);
}

// tile index of (rb, cb), 1 <= cb <= rb <= nbk (block row nbk = right-hand side), column-major over cb
__device__ __forceinline__ int df_tile_index(int rb, int cb, int nbk)
{
    // tiles of columns 1 .. cb-1: sum_{c=1}^{cb-1} (nbk - c + 1)
    const int before = (cb - 1) * (nbk + 1) - (cb - 1) * cb / 2;
    return before + (rb - cb);
}

// dev-only accounting of CTA 0, thread 0 (read and reset by bsfm_debug_df_prof): [0] kernel ns, [1] potf2, [2] up to the barrier
// behind inverse + loads, [3] X Z^T strips -- BAR.SYNC defers its blocking to the first dependent instruction, so the WAIT for the
// look-ahead inputs shows up here --, [4] factor block out + update of the next diagonal tile, [5] end-of-step barrier, [6] steps,
// [7] launches   ([1..5] in SM cycles)
// They stay because the kernel is faster with them: without the clock reads a 450 x 450 factorisation took 166 us instead of
// 159 us (H100 80GB HBM3, 400 W power limit), and empty compiler fences at the same points did not recover it.
__device__ unsigned long long g_df_prof[8];
__device__ __forceinline__ unsigned long long df_clock() { unsigned long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) :: "memory"); return t; }
__device__ __forceinline__ unsigned long long df_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory"); return t; }

// named barriers of CTA 0 (0 = __syncthreads, 2..5 = potf2 panels, see ba_chol_potf2.cuh)
#define DF_BAR(id, count) asm volatile("bar.sync %0, %1;" ::"n"(id), "n"(count) : "memory")
#define DF_ARRIVE(id, count) asm volatile("bar.arrive %0, %1;" ::"n"(id), "n"(count) : "memory")

__global__ void __launch_bounds__(DF_THREADS, 1) chol_dataflow_kernel(const double *A, double *Lout, int ld, int n, double *linv_all /* pre-filled */,
                                                                     double *Pub /* (n + 1) x ldp finished tiles, pre-filled */, int ldp, Scalars *sc)
{
    __shared__ __align__(16) double tiles[5][LNB][TP];      // CTA 0: L_kk, next diagonal tile, X, Z, W;  workers: Z, 2 x (X_r, X_c)
    __shared__ double dinv[LNB];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;
    const int nbk = (n + LNB - 1) / LNB;
    const int workers = (int) gridDim.x - 1;

    auto rows_of = [&](int rb) { return (rb == nbk) ? 1 : min(LNB, n - rb * LNB); };
    auto rbase_of = [&](int rb) { return (rb == nbk) ? n : rb * LNB; };

    if (blockIdx.x == 0) {
        // ================= the diagonal chain =================
        // per 32-column step k:
        //   warp 0       potf2 of the diagonal tile (warp_potf2_32_tc)          warp 1   its inverse Z_kk, one panel behind
        //   warps 2, 3   fetch the look-ahead inputs -- sub-diagonal block (k+1, k) and diagonal tile (k+1, k+1), both finished by
        //                their owners with step k-1 -- as soon as their words arrive
        //   warps 4..7   send Z_kk out the moment warps 0 / 1 are done (they never wait for the loads), then L_kk
        //   warps 0..3   X <- X Z^T for the sub-diagonal block, rank-32 update of the next diagonal tile, which never leaves
        //                shared memory
        double (*Lc)[TP] = tiles[0], (*Ln)[TP] = tiles[1];
        double (*Xr)[TP] = tiles[2], (*Zs)[TP] = tiles[3], (*Ws)[TP] = tiles[4];
        const unsigned long long ns0 = df_ns();
        unsigned long long pc[5] = {0, 0, 0, 0, 0}, tc = 0;
        {
            const int nb0 = min(LNB, n);
            for (int e = tid; e < LNB * LNB; e += DF_THREADS) {
                const int r = e >> 5, c = e & 31;
                Lc[r][c] = (r < nb0 && c <= r) ? A[(size_t) r * ld + c] : ((r == c) ? 1.0 : 0.0);
                Zs[r][c] = 0.0;                              // the strictly upper blocks of Z stay zero
            }
        }
        __syncthreads();
        for (int k = 0; k < nbk; k++) {
            const int k0 = k * LNB, nb = min(LNB, n - k0);
            const bool last = (k + 1 == nbk);
            const int rb = last ? nbk : k + 1;                 // last step: the right-hand side segment instead of a diagonal tile
            const int rrows = rows_of(rb), rbase = rbase_of(rb);
            tc = df_clock();
            if (warp >= 4) {
                // ---- senders ----
                DF_BAR(7, 192);                                 // potf2 and inverse done
                for (int e = tid - 128; e < LNB * LNB; e += 128) st_strong(&linv_all[(size_t) k * LNB * LNB + e], ((e & 31) <= (e >> 5)) ? Zs[e >> 5][e & 31] : 0.0);
                for (int e = tid - 128; e < LNB * LNB; e += 128) {
                    const int r = e >> 5, c = e & 31;
                    if (r < nb && c <= r) Lout[(size_t) (k0 + r) * ld + (k0 + c)] = Lc[r][c];
                }
            } else {
                if (warp == 0) {
                    const bool bad = warp_potf2_32_tc(Lc, dinv, lane, true);
                    if (bad && lane == 0) sc->chol_fail = 1;
                    __syncwarp();
                    { const unsigned long long t = df_clock(); pc[0] += t - tc; tc = t; }
                    DF_ARRIVE(7, 192);
                } else if (warp == 1) {
                    warp_tile_inverse(Lc, dinv, Zs, Ws, lane);
                    DF_ARRIVE(7, 192);
                } else {
                    const double *src = (k == 0) ? A : Pub;     // step 0 reads the untouched input
                    const int lds = (k == 0) ? ld : ldp;
                    const int t64 = tid - 64;
#pragma unroll 1
                    for (int e0 = 0; e0 < LNB * LNB; e0 += 64 * 8) {
                        df_fetch<8>([&](int i) -> const double * { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                                   return (r < rrows && c < nb) ? &src[(size_t) (rbase + r) * lds + (k0 + c)] : nullptr; },
                                    [&](int i, double v) { const int e = e0 + t64 + 64 * i; Xr[e >> 5][e & 31] = v; }, sc);
                        if (!last)
                            df_fetch<8>([&](int i) -> const double * { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                                       return (r < rrows && c <= r) ? &src[(size_t) (rbase + r) * lds + (rbase + c)] : nullptr; },
                                        [&](int i, double v) { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                               Ln[r][c] = (r < rrows && c <= r) ? v : ((r == c) ? 1.0 : 0.0); }, sc);
                    }
                }
                DF_BAR(8, 128);                                 // factor, inverse and look-ahead inputs are in shared memory
                { const unsigned long long t = df_clock(); pc[1] += t - tc; tc = t; }
                warp_rows_times_ZT(Xr, 8 * warp, Zs, lane);
                DF_BAR(8, 128);
                { const unsigned long long t = df_clock(); pc[2] += t - tc; tc = t; }
                for (int e = tid; e < LNB * LNB; e += 128) {
                    const int r = e >> 5, c = e & 31;
                    if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
                }
                if (!last) {
                    for (int t = warp; t < 10; t += 4) {       // lower 8 x 8 tiles (ri, cj)
                        int ri = 0, rem = t;
                        while (rem > ri) { rem -= ri + 1; ri++; }
                        const int cj = rem;
                        double c0 = 0.0, c1 = 0.0;
#pragma unroll
                        for (int ks = 0; ks < LNB; ks += 4) tile_dmma(c0, c1, Xr[8 * ri + g][ks + tg], Xr[8 * cj + g][ks + tg]);
                        double2 cur = *reinterpret_cast<const double2 *>(&Ln[8 * ri + g][8 * cj + 2 * tg]);
                        cur.x -= c0; cur.y -= c1;
                        *reinterpret_cast<double2 *>(&Ln[8 * ri + g][8 * cj + 2 * tg]) = cur;
                    }
                }
                { const unsigned long long t = df_clock(); pc[3] += t - tc; tc = t; }
            }
            __syncthreads();
            { const unsigned long long t = df_clock(); pc[4] += t - tc; tc = t; }
            double (*tmp)[TP] = Lc; Lc = Ln; Ln = tmp;
        }
        if (tid == 0) {
            g_df_prof[0] += df_ns() - ns0;
            for (int i = 0; i < 5; i++) g_df_prof[1 + i] += pc[i];
            g_df_prof[6] += nbk;
            g_df_prof[7] += 1;
        }
        return;
    }

    // ================= workers: static tile ownership, the owned tiles live in REGISTERS =================
    // Tile (rb, cb) (1 <= cb < nbk, cb <= rb <= nbk; row block nbk = right-hand side) takes the rank-32 updates of steps
    // k = 0 .. klast (klast = cb - 1; cb - 2 for a diagonal tile, whose step cb - 1 is CTA 0's look-ahead) and is read by other CTAs
    // only after that: it goes out to `Pub` exactly once.  Each CTA owns at most two tiles (DMMA accumulator layout: warp w holds
    // the 8 x 8 sub-tiles 2 w, 2 w + 1).  Per step: fetch the two panel blocks of every owned tile (finished with step k - 1), then
    // Z_kk, then X <- X Z^T strips and the update, all on the fp64 tensor cores.
    double (*Zs)[TP] = tiles[0];
    const int w = (int) blockIdx.x - 1;
    int ntile = 0;
    for (int c = 1; c < nbk; c++) ntile += nbk - c + 1;
    int trb[2], tcb[2], klast[2];
    double cur[2][2][2];
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const int ti = w + s * workers;
        trb[s] = tcb[s] = 0; klast[s] = -1;
        if (ti < ntile) {
            int c = 1, rem = ti;
            while (rem >= nbk - c + 1) { rem -= nbk - c + 1; c++; }
            tcb[s] = c; trb[s] = c + rem;
            klast[s] = (trb[s] == c) ? c - 2 : c - 1;
        }
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int t = warp * 2 + i, r = 8 * (t >> 2) + g, c = 8 * (t & 3) + 2 * tg;
            cur[s][i][0] = cur[s][i][1] = 0.0;
            if (klast[s] >= 0) {
                const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]);
                const double *src = &A[(size_t) (rbase_of(trb[s]) + r) * ld + (tcb[s] * LNB + c)];
                if (r < rrows && c < crows) cur[s][i][0] = src[0];
                if (r < rrows && c + 1 < crows) cur[s][i][1] = src[1];
            }
        }
    }
    const int kend = max(klast[0], klast[1]);
    for (int k = 0; k <= kend; k++) {
        const int k0 = k * LNB, nb = min(LNB, n - k0);
        const double *src = (k == 0) ? A : Pub;
        const int lds = (k == 0) ? ld : ldp;
        // (a) the panel blocks of the owned tiles: finished by their owners with step k - 1
#pragma unroll
        for (int s = 0; s < 2; s++) {
            if (k > klast[s]) continue;
            double (*Xr)[TP] = tiles[1 + 2 * s], (*Xc)[TP] = tiles[2 + 2 * s];
            const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]), rbase = rbase_of(trb[s]), cbase = tcb[s] * LNB;
            df_fetch<4>([&](int i) -> const double * { const int e = tid + DF_THREADS * i, r = e >> 5, c = e & 31;
                                                       return (r < rrows && c < nb) ? &src[(size_t) (rbase + r) * lds + (k0 + c)] : nullptr; },
                        [&](int i, double v) { const int e = tid + DF_THREADS * i; Xr[e >> 5][e & 31] = v; }, sc);
            if (trb[s] != tcb[s])
                df_fetch<4>([&](int i) -> const double * { const int e = tid + DF_THREADS * i, r = e >> 5, c = e & 31;
                                                           return (r < crows && c < nb) ? &src[(size_t) (cbase + r) * lds + (k0 + c)] : nullptr; },
                            [&](int i, double v) { const int e = tid + DF_THREADS * i; Xc[e >> 5][e & 31] = v; }, sc);
        }
        // (b) Z_kk
        df_fetch<4>([&](int i) -> const double * { return &linv_all[(size_t) k * LNB * LNB + tid + DF_THREADS * i]; },
                    [&](int i, double v) { const int e = tid + DF_THREADS * i; Zs[e >> 5][e & 31] = v; }, sc);
        __syncthreads();
        // (c) X <- X Z^T: up to 16 eight-row strips, two per warp
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int which = (warp >> 2) & 1, strip = warp & 3;          // slot j: warps 0..3 its row block, warps 4..7 its column block
            if (k > klast[j] || (which == 1 && trb[j] == tcb[j])) continue;
            warp_rows_times_ZT(tiles[1 + 2 * j + which], 8 * strip, Zs, lane);
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < 2; s++) {
            if (k > klast[s]) continue;
            const double (*Xr)[TP] = tiles[1 + 2 * s];
            const double (*XC)[TP] = (trb[s] != tcb[s]) ? tiles[2 + 2 * s] : tiles[1 + 2 * s];
            const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]), rbase = rbase_of(trb[s]), cbase = tcb[s] * LNB;
            // (e) tile -= X_r X_c^T
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int t = warp * 2 + i, ri = t >> 2, cj = t & 3;
                double a0 = 0.0, a1 = 0.0;
#pragma unroll
                for (int ks = 0; ks < LNB; ks += 4) tile_dmma(a0, a1, Xr[8 * ri + g][ks + tg], XC[8 * cj + g][ks + tg]);
                cur[s][i][0] -= a0; cur[s][i][1] -= a1;
            }
            // (f) finished: out to the other CTAs, once (the words are their own flags)
            if (k == klast[s]) {
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const int t = warp * 2 + i, r = 8 * (t >> 2) + g, c = 8 * (t & 3) + 2 * tg;
                    double *dst = &Pub[(size_t) (rbase + r) * ldp + (cbase + c)];
                    const bool dg = (trb[s] == tcb[s]);                 // diagonal tile: lower triangle only
                    if (r < rrows && c < crows && (!dg || c <= r)) st_strong(dst, cur[s][i][0]);
                    if (r < rrows && c + 1 < crows && (!dg || c + 1 <= r)) st_strong(dst + 1, cur[s][i][1]);
                }
            }
            if (tcb[s] == k + 1) {          // first column: this tile's row block of the factor (read by the back substitution only)
                for (int e = tid; e < LNB * LNB; e += DF_THREADS) {
                    const int r = e >> 5, c = e & 31;
                    if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
                }
            }
        }
        __syncthreads();                    // the X buffers are free again
    }
}

// ================= the same dataflow over the envelope of a large banded system =================
// chol_band_kernel factors a system whose rows have a narrow envelope (CholBandPlan, ba_chol_large.cuh) in one cooperative
// launch; the tiles outside the envelope are zero in L and never touched.
//   CTA 0        the diagonal chain of chol_dataflow_kernel, except that the sub-diagonal block (k+1, k) may lie outside the
//                envelope (it is zero then: no look-ahead update), and the sender warp 4 forms the right-hand-side segment
//                y_k = (row n, block k) Z_kk^T at every step
//   CTAs 1..W    the tiles of the host's schedule, at most two at a time in registers: a tile enters its slot from A at its
//                first update step and leaves through the publish buffer after its last.  A worker fetches panel blocks and
//                Z_kk only at the steps where one of its tiles takes an update.  The owner of a diagonal tile (rb, rb) writes
//                block (rb, k) of L at every step k it takes, which covers every envelope block below the sub-diagonal.
//   publish      envelope-packed: tile (rb, cb) is the 32 x 32 block number toff[rb] + cb - env[rb] (row pitch 32).  A tile that
//                took no update from a worker is read from A by its consumers.
__global__ void __launch_bounds__(DF_THREADS, 1) chol_band_kernel(const double *A, double *Lout, int ld, int n, double *linv_all /* pre-filled */,
                                                                  double *Pub /* pre-filled */, const CholBand B, long long spin_limit, Scalars *sc)
{
    __shared__ __align__(16) double tiles[5][LNB][TP];      // CTA 0: L_kk, next diagonal tile, X, Z, W;  workers: Z, 2 x (X_r, X_c)
    __shared__ __align__(16) double yrow[8][TP];            // CTA 0: the right-hand-side segment in row 0 (rows 1..7 stay zero)
    __shared__ double dinv[LNB];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;
    const int nbk = (n + LNB - 1) / LNB;
    const int *env = B.env;

    auto rows_of = [&](int rb) { return (rb == nbk) ? 1 : min(LNB, n - rb * LNB); };
    auto rbase_of = [&](int rb) { return (rb == nbk) ? n : rb * LNB; };
    // finished envelope tile (x, c): element (r, q) is p[r * lds + q]
    struct TileSrc { const double *p; int lds; };
    auto tile_src = [&](int x, int c) -> TileSrc {
        const bool worked = max(env[x], env[c]) <= ((x == c) ? c - 2 : c - 1);
        if (worked) return {Pub + ((size_t) (B.toff[x] + c - env[x]) << 10), LNB};
        return {A + (size_t) rbase_of(x) * ld + (size_t) c * LNB, ld};
    };

    if (blockIdx.x == 0) {
        double (*Lc)[TP] = tiles[0], (*Ln)[TP] = tiles[1];
        double (*Xr)[TP] = tiles[2], (*Zs)[TP] = tiles[3], (*Ws)[TP] = tiles[4];
        {
            const int nb0 = min(LNB, n);
            for (int e = tid; e < LNB * LNB; e += DF_THREADS) {
                const int r = e >> 5, c = e & 31;
                Lc[r][c] = (r < nb0 && c <= r) ? A[(size_t) r * ld + c] : ((r == c) ? 1.0 : 0.0);
                Zs[r][c] = 0.0;
            }
            for (int e = tid; e < 8 * TP; e += DF_THREADS) yrow[e / TP][e % TP] = 0.0;
        }
        __syncthreads();
        for (int k = 0; k < nbk; k++) {
            const int k0 = k * LNB, nb = min(LNB, n - k0);
            const bool last = (k + 1 == nbk);
            const bool sub = !last && env[k + 1] <= k;          // block (k+1, k) lies in the envelope
            const int rrows = last ? 0 : rows_of(k + 1), rbase = (k + 1) * LNB;
            if (warp >= 4) {
                // ---- senders ----
                DF_BAR(7, 192);                                 // potf2 and inverse done
                for (int e = tid - 128; e < LNB * LNB; e += 128) st_strong(&linv_all[(size_t) k * LNB * LNB + e], ((e & 31) <= (e >> 5)) ? Zs[e >> 5][e & 31] : 0.0);
                for (int e = tid - 128; e < LNB * LNB; e += 128) {
                    const int r = e >> 5, c = e & 31;
                    if (r < nb && c <= r) Lout[(size_t) (k0 + r) * ld + (k0 + c)] = Lc[r][c];
                }
                if (warp == 4) {                                // forward substitution: y_k, after Z_kk has gone out
                    const TileSrc y = tile_src(nbk, k);
                    df_fetch<1>([&](int) -> const double * { return (lane < nb) ? y.p + lane : nullptr; },
                                [&](int, double v) { yrow[0][lane] = v; }, sc, spin_limit);
                    __syncwarp();
                    warp_rows_times_ZT(yrow, 0, Zs, lane);
                    __syncwarp();
                    if (lane < nb) Lout[(size_t) n * ld + (k0 + lane)] = yrow[0][lane];
                }
            } else {
                if (warp == 0) {
                    const bool bad = warp_potf2_32_tc(Lc, dinv, lane, true);
                    if (bad && lane == 0) sc->chol_fail = 1;
                    __syncwarp();
                    DF_ARRIVE(7, 192);
                } else if (warp == 1) {
                    warp_tile_inverse(Lc, dinv, Zs, Ws, lane);
                    DF_ARRIVE(7, 192);
                } else if (!last) {
                    const TileSrc xs = sub ? tile_src(k + 1, k) : TileSrc{A, ld};
                    const TileSrc ds = tile_src(k + 1, k + 1);
                    const int t64 = tid - 64;
#pragma unroll 1
                    for (int e0 = 0; e0 < LNB * LNB; e0 += 64 * 8) {
                        if (sub)
                            df_fetch<8>([&](int i) -> const double * { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                                       return (r < rrows && c < nb) ? xs.p + (size_t) r * xs.lds + c : nullptr; },
                                        [&](int i, double v) { const int e = e0 + t64 + 64 * i; Xr[e >> 5][e & 31] = v; }, sc, spin_limit);
                        df_fetch<8>([&](int i) -> const double * { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                                   return (r < rrows && c <= r) ? ds.p + (size_t) r * ds.lds + c : nullptr; },
                                    [&](int i, double v) { const int e = e0 + t64 + 64 * i, r = e >> 5, c = e & 31;
                                                           Ln[r][c] = (r < rrows && c <= r) ? v : ((r == c) ? 1.0 : 0.0); }, sc, spin_limit);
                    }
                }
                DF_BAR(8, 128);                                 // factor, inverse and look-ahead inputs are in shared memory
                if (sub) warp_rows_times_ZT(Xr, 8 * warp, Zs, lane);
                DF_BAR(8, 128);
                if (sub) {
                    for (int e = tid; e < LNB * LNB; e += 128) {
                        const int r = e >> 5, c = e & 31;
                        if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
                    }
                    for (int t = warp; t < 10; t += 4) {       // lower 8 x 8 tiles (ri, cj) of the next diagonal tile
                        int ri = 0, rem = t;
                        while (rem > ri) { rem -= ri + 1; ri++; }
                        const int cj = rem;
                        double c0 = 0.0, c1 = 0.0;
#pragma unroll
                        for (int ks = 0; ks < LNB; ks += 4) tile_dmma(c0, c1, Xr[8 * ri + g][ks + tg], Xr[8 * cj + g][ks + tg]);
                        double2 cur = *reinterpret_cast<const double2 *>(&Ln[8 * ri + g][8 * cj + 2 * tg]);
                        cur.x -= c0; cur.y -= c1;
                        *reinterpret_cast<double2 *>(&Ln[8 * ri + g][8 * cj + 2 * tg]) = cur;
                    }
                }
            }
            __syncthreads();
            double (*tmp)[TP] = Lc; Lc = Ln; Ln = tmp;
        }
        return;
    }

    // ================= workers: the host's schedule, two register slots =================
    double (*Zs)[TP] = tiles[0];
    const int w = (int) blockIdx.x - 1;
    constexpr int NONE = 0x7fffffff;
    int next[2], stop[2], trb[2], tcb[2], klast[2], knext[2];
    double cur[2][2][2];
    auto take = [&](int s) {        // the slot's next tile (knext = its first update step), its values from A
        trb[s] = tcb[s] = 0; klast[s] = -1; knext[s] = NONE;
        if (next[s] < stop[s]) {
            const int t = B.sched[next[s]];
            trb[s] = t >> 16; tcb[s] = t & 0xffff;
            knext[s] = max(env[trb[s]], env[tcb[s]]);
            klast[s] = (trb[s] == tcb[s]) ? tcb[s] - 2 : tcb[s] - 1;
        }
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int t = warp * 2 + i, r = 8 * (t >> 2) + g, c = 8 * (t & 3) + 2 * tg;
            cur[s][i][0] = cur[s][i][1] = 0.0;
            if (knext[s] != NONE) {
                const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]);
                const double *src = &A[(size_t) (rbase_of(trb[s]) + r) * ld + (tcb[s] * LNB + c)];
                if (r < rrows && c < crows) cur[s][i][0] = src[0];
                if (r < rrows && c + 1 < crows) cur[s][i][1] = src[1];
            }
        }
    };
#pragma unroll
    for (int s = 0; s < 2; s++) {
        next[s] = B.sptr[2 * w + s]; stop[s] = B.sptr[2 * w + s + 1];
        take(s);
    }
    while (true) {
        const int k = min(knext[0], knext[1]);
        if (k == NONE) break;
        const int k0 = k * LNB, nb = min(LNB, n - k0);
        // (a) the panel blocks of the tiles updated at this step: finished with step k - 1
#pragma unroll
        for (int s = 0; s < 2; s++) {
            if (knext[s] != k) continue;
            double (*Xr)[TP] = tiles[1 + 2 * s], (*Xc)[TP] = tiles[2 + 2 * s];
            const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]);
            const TileSrc rs = tile_src(trb[s], k);
            df_fetch<4>([&](int i) -> const double * { const int e = tid + DF_THREADS * i, r = e >> 5, c = e & 31;
                                                       return (r < rrows && c < nb) ? rs.p + (size_t) r * rs.lds + c : nullptr; },
                        [&](int i, double v) { const int e = tid + DF_THREADS * i; Xr[e >> 5][e & 31] = v; }, sc, spin_limit);
            if (trb[s] != tcb[s]) {
                const TileSrc cs = tile_src(tcb[s], k);
                df_fetch<4>([&](int i) -> const double * { const int e = tid + DF_THREADS * i, r = e >> 5, c = e & 31;
                                                           return (r < crows && c < nb) ? cs.p + (size_t) r * cs.lds + c : nullptr; },
                            [&](int i, double v) { const int e = tid + DF_THREADS * i; Xc[e >> 5][e & 31] = v; }, sc, spin_limit);
            }
        }
        // (b) Z_kk
        df_fetch<4>([&](int i) -> const double * { return &linv_all[(size_t) k * LNB * LNB + tid + DF_THREADS * i]; },
                    [&](int i, double v) { const int e = tid + DF_THREADS * i; Zs[e >> 5][e & 31] = v; }, sc, spin_limit);
        __syncthreads();
        // (c) X <- X Z^T: up to 16 eight-row strips, two per warp
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int which = (warp >> 2) & 1, strip = warp & 3;
            if (knext[j] != k || (which == 1 && trb[j] == tcb[j])) continue;
            warp_rows_times_ZT(tiles[1 + 2 * j + which], 8 * strip, Zs, lane);
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < 2; s++) {
            if (knext[s] != k) continue;
            const double (*Xr)[TP] = tiles[1 + 2 * s];
            const bool dg = (trb[s] == tcb[s]);
            const double (*XC)[TP] = dg ? tiles[1 + 2 * s] : tiles[2 + 2 * s];
            const int rrows = rows_of(trb[s]), crows = rows_of(tcb[s]), rbase = rbase_of(trb[s]);
            // (d) tile -= X_r X_c^T
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int t = warp * 2 + i, ri = t >> 2, cj = t & 3;
                double a0 = 0.0, a1 = 0.0;
#pragma unroll
                for (int ks = 0; ks < LNB; ks += 4) tile_dmma(a0, a1, Xr[8 * ri + g][ks + tg], XC[8 * cj + g][ks + tg]);
                cur[s][i][0] -= a0; cur[s][i][1] -= a1;
            }
            // (e) finished: into the publish buffer, once (the words are their own flags)
            if (k == klast[s]) {
                double *dst = Pub + ((size_t) (B.toff[trb[s]] + tcb[s] - env[trb[s]]) << 10);
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const int t = warp * 2 + i, r = 8 * (t >> 2) + g, c = 8 * (t & 3) + 2 * tg;
                    if (r < rrows && c < crows && (!dg || c <= r)) st_strong(&dst[r * LNB + c], cur[s][i][0]);
                    if (r < rrows && c + 1 < crows && (!dg || c + 1 <= r)) st_strong(&dst[r * LNB + c + 1], cur[s][i][1]);
                }
            }
            // (f) a diagonal tile's owner writes block (rb, k) of the factor (read by the back substitution only)
            if (dg) {
                for (int e = tid; e < LNB * LNB; e += DF_THREADS) {
                    const int r = e >> 5, c = e & 31;
                    if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
                }
            }
        }
        __syncthreads();                    // the X buffers are free again
#pragma unroll
        for (int s = 0; s < 2; s++) {
            if (knext[s] != k) continue;
            if (k == klast[s]) { next[s]++; take(s); }
            else knext[s] = k + 1;
        }
    }
}

// Back substitution L^T x = y over the envelope, one CTA: y (row n of the factor) in shared memory; step kb reads the columns
// [32 env[kb], 32 kb) of its 32 factor rows only.  Same arithmetic per step as chol_backsolve_blocked_kernel.
__global__ void __launch_bounds__(512) chol_backsolve_band_kernel(const double *L, int ld, int n, const double *Linv_all, const int *env, double *x)
{
    extern __shared__ double ys[];      // n
    __shared__ double xk[LNB];
    __shared__ double Li[LNB][LNB + 1];
    const int tid = threadIdx.x;
    const double *yrow = L + (size_t) n * ld;
    for (int c = tid; c < n; c += 512) ys[c] = yrow[c];
    const int nbk = (n + LNB - 1) / LNB;
    // the inverse block and this thread's column of the factor rows of step kb - 1 are fetched one step ahead
    double z0, z1, l[LNB];
    {
        const int kb = nbk - 1, k0 = kb * LNB, nb = min(LNB, n - k0), c = LNB * env[kb] + tid;
        z0 = Linv_all[(size_t) kb * LNB * LNB + tid]; z1 = Linv_all[(size_t) kb * LNB * LNB + 512 + tid];
#pragma unroll
        for (int r = 0; r < LNB; r++) l[r] = (c < k0 && r < nb) ? L[(size_t) (k0 + r) * ld + c] : 0.0;
    }
    for (int kb = nbk - 1; kb >= 0; kb--) {
        const int k0 = kb * LNB, nb = min(LNB, n - k0), e0 = LNB * env[kb];
        Li[tid >> 5][tid & 31] = z0;
        Li[16 + (tid >> 5)][tid & 31] = z1;
        if (kb > 0) { z0 = Linv_all[(size_t) (kb - 1) * LNB * LNB + tid]; z1 = Linv_all[(size_t) (kb - 1) * LNB * LNB + 512 + tid]; }
        __syncthreads();
        // x_k = L_kk^-T y_k : 8 lanes per output, 4 terms each, shuffle-reduced
        if (tid < 256) {
            const int o = tid >> 3, part = tid & 7;
            double sacc = 0.0;
#pragma unroll
            for (int u = 0; u < 4; u++) { const int r = part * 4 + u; if (r >= o && r < nb) sacc = fma(Li[r][o], ys[k0 + r], sacc); }
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 1);
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 2);
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 4);
            if (part == 0) { xk[o] = sacc; if (o < nb) x[k0 + o] = sacc; }
        }
        __syncthreads();
        if (e0 + tid < k0) {
            double sacc = 0.0;
#pragma unroll
            for (int r = 0; r < LNB; r++) sacc = fma(l[r], xk[r], sacc);
            ys[e0 + tid] -= sacc;
        }
        for (int c = e0 + tid + 512; c < k0; c += 512) {      // envelopes wider than 512 columns: 16 rows at a time
            double sacc = 0.0;
#pragma unroll 1
            for (int r0 = 0; r0 < LNB; r0 += 16) {
                double lv[16];
#pragma unroll
                for (int r = 0; r < 16; r++) lv[r] = (r0 + r < nb) ? L[(size_t) (k0 + r0 + r) * ld + c] : 0.0;
#pragma unroll
                for (int r = 0; r < 16; r++) sacc = fma(lv[r], xk[r0 + r], sacc);
            }
            ys[c] -= sacc;
        }
        if (kb > 0) {                       // rows of step kb - 1 (a full block)
            const int k1 = k0 - LNB, c = LNB * env[kb - 1] + tid;
#pragma unroll
            for (int r = 0; r < LNB; r++) l[r] = (c < k1) ? L[(size_t) (k1 + r) * ld + c] : 0.0;
        }
    }
}

int chol_band_factor(cudaStream_t st, const double *A, double *Lmat, int n, double *linv_ws, const CholBand &B, Scalars *sc)
{
    const int nbk = (n + LNB - 1) / LNB;
    if ((size_t) B.ntile > chol_band_capacity_tiles(n) || n > CHOL_BAND_MAX_N || B.workers < 1) {
        set_error("chol_band_factor: the plan of n = %d does not fit the workspace", n);
        return BSFM_ERR_ARG;
    }
    // the Z blocks and the packed publish buffer right behind them (in the panel path's xinv area, unused here) are pre-filled
    // with the "not yet" pattern in one memset
    double *pub = linv_ws + (size_t) nbk * LNB * LNB;
    BSFM_CUDA_TRY(cudaMemsetAsync(linv_ws, 0xFF, ((size_t) nbk + B.ntile) * LNB * LNB * sizeof(double), st));
    long long spin_limit = DF_SPIN_LIMIT + (long long) nbk * DF_SPIN_PER_STEP;
    int ld = n;
    CholBand b = B;
    void *args[] = {&A, &Lmat, &ld, &n, &linv_ws, &pub, &b, &spin_limit, &sc};
    BSFM_CUDA_TRY(cudaLaunchCooperativeKernel((const void *) chol_band_kernel, dim3(1 + B.workers), dim3(DF_THREADS), args, 0, st));
    count_launch();
    return BSFM_OK;
}

int chol_band_backsolve(cudaStream_t st, const double *Lmat, int n, const double *linv_ws, const CholBand &B, double *x)
{
    int dev = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    static std::atomic<int> attr_set[64];
    if (dev >= 0 && dev < 64 && !attr_set[dev].load()) {
        BSFM_CUDA_TRY(cudaFuncSetAttribute(chol_backsolve_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) (CHOL_BAND_MAX_N * sizeof(double))));
        attr_set[dev].store(1);
    }
    chol_backsolve_band_kernel<<<1, 512, (size_t) n * sizeof(double), st>>>(Lmat, n, n, linv_ws, B.env, x);
    BSFM_KERNEL_CHECK();
    return BSFM_OK;
}

__global__ void __launch_bounds__(512) chol_backsolve_blocked_kernel(const double *A, int ld, int n, const double *Linv_all, double *x, double *ywork);

// Factorisation only: A (pitch ld, n x n lower + right-hand side row n) -> Lmat (same pitch), inverses of the 32 x 32 diagonal blocks
// -> linv_blocks[k * 1024].  pub: (n + 1) x n doubles of scratch.  A and Lmat may point INTO a larger matrix (the large path
// finishes its last panels with this kernel).  *used = false: not usable here (caller falls back), nothing launched.
int chol_dataflow_factor(cudaStream_t st, const double *A, double *Lmat, int ld, int n, double *linv_blocks, double *pub, Scalars *sc, bool *used)
{
    *used = false;
    static const bool enabled = []() { const char *e = getenv("BSFM_BA_CHOL_DATAFLOW"); return !(e && e[0] == '0'); }();
    if (!enabled) return BSFM_OK;
    int dev = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    static std::atomic<int> coop_ok[64];      // 0 unknown, 1 yes, -1 no
    static std::atomic<int> sm_count[64];
    if (dev < 0 || dev >= 64) return BSFM_OK;
    if (coop_ok[dev].load() == 0) {
        int coop = 0, sms = 0;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        sm_count[dev].store(sms);
        coop_ok[dev].store(coop ? 1 : -1);
    }
    if (coop_ok[dev].load() != 1) return BSFM_OK;
    const int nbk = (n + LNB - 1) / LNB;
    if (nbk < 2 || nbk > DF_MAX_NBK || n > DF_MAX_N) return BSFM_OK;      // larger systems: more than two tiles per worker
    int ntile = 0;
    for (int c = 1; c < nbk; c++) ntile += nbk - c + 1;
    const int grid = std::min(sm_count[dev].load(), 1 + std::max(1, ntile));
    if (grid < 2 || ntile > 2 * (grid - 1)) return BSFM_OK;      // every worker keeps at most two tiles in registers
    // the Z blocks and the tile area are pre-filled with the "not yet" pattern (all ones): one memset when they are one range
    const size_t zbytes = (size_t) nbk * LNB * LNB * sizeof(double), pbytes = (size_t) (n + 1) * n * sizeof(double);
    const char *zb = reinterpret_cast<const char *>(linv_blocks), *pb = reinterpret_cast<const char *>(pub);
    if (pb >= zb + zbytes && (size_t) (pb - zb) <= zbytes + (1u << 20)) {
        BSFM_CUDA_TRY(cudaMemsetAsync(linv_blocks, 0xFF, (size_t) (pb - zb) + pbytes, st));
    } else {
        BSFM_CUDA_TRY(cudaMemsetAsync(linv_blocks, 0xFF, zbytes, st));
        BSFM_CUDA_TRY(cudaMemsetAsync(pub, 0xFF, pbytes, st));
    }
    int ldp = n;
    void *args[] = {&A, &Lmat, &ld, &n, &linv_blocks, &pub, &ldp, &sc};
    BSFM_CUDA_TRY(cudaLaunchCooperativeKernel((const void *) chol_dataflow_kernel, dim3(grid), dim3(DF_THREADS), args, 0, st));
    count_launch();
    *used = true;
    return BSFM_OK;
}

// small systems: factorisation + back substitution.  linv_ws: [Z blocks nbk x 1024][back-substitution scratch n + 64][(n + 1) x n]
int chol_solve_dataflow(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *x, Scalars *sc, bool *used)
{
    const int nbk = (n + LNB - 1) / LNB;
    double *ywork = linv_ws + (size_t) nbk * LNB * LNB;
    int rc = chol_dataflow_factor(st, A, Lmat, n, n, linv_ws, ywork + n + 64, sc, used);
    if (rc != BSFM_OK || !*used) return rc;
    chol_backsolve_blocked_kernel<<<1, 512, 0, st>>>(Lmat, n, n, linv_ws, x, ywork);
    BSFM_KERNEL_CHECK();
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm

// dev-only: read and reset chol_dataflow_kernel's CTA-0 counters (see g_df_prof)
extern "C" int bsfm_debug_df_prof(unsigned long long *out8)
{
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemcpyFromSymbol(out8, bsfm::ba::g_df_prof, 8 * sizeof(unsigned long long)) != cudaSuccess) return -1;
    unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    return cudaMemcpyToSymbol(bsfm::ba::g_df_prof, z, sizeof(z)) == cudaSuccess ? 0 : -1;
}
