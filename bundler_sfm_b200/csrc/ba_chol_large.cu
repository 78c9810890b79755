// ba_chol_large.cu -- dense SPD solve of LARGE reduced camera systems (n > 1536; config 3: 1000 cameras -> 9000^2).
// Reference: sba_Axb_Chol = LAPACK dpotrf + dpotrs, lib/sba-1.5/sba_lapack.c:374-485.
//
// Right-looking blocked Cholesky (lower, row-major, factor OUT OF PLACE in Lmat, right-hand side carried as matrix
// row n so the forward substitution falls out of the panel solves), outer panels of 256 columns, FOUR launches per
// panel:
//   chol_diag_kernel      1 CTA : fp64 factorisation of the 256 x 256 diagonal block (32-column sub-steps: one warp
//                                 factors the 32 x 32 block in REGISTERS with shuffles, thread-per-row solves, rank-32
//                                 in-block update) + the inverses of its eight 32 x 32 diagonal sub-blocks
//   chol_trsm_kernel      64 rows x 256 columns per CTA : L_panel = A_panel L_kk^-T as a blocked forward substitution
//                                 (small GEMMs against the sub-block inverses)
//   chol_syrk_dmma_kernel A -= L_panel L_panel^T, K = 256, on the fp64 tensor cores: persistent, warp-specialised, fed
//                                 by TMA from a pre-tiled image of the panel that chol_trsm_kernel writes
//   (after the last panel) chol_backsolve_big_kernel per panel, last to first: L^T x = y
// The small-system path (ba_chol.cu: one fused launch per 32 columns) stays as it is: it is latency-bound, this one is
// throughput-bound.
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"
#include "ba_chol_potf2.cuh"
#include "common.h"
#include "tc_ptx.cuh"
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <vector>

namespace bsfm {
namespace ba {

// fp64 tensor-core tile product (DMMA): D(8x8) += A(8x4) B(4x8); lane = 4 g + tg holds A[g][tg], B[tg][g] (= B^T[g][tg]),
// D[g][2 tg], D[g][2 tg + 1]
__device__ __forceinline__ void dmma_m8n8k4(double &d0, double &d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// ---- 256 x 256 diagonal block ----------------------------------------------------------------------------------
// One CTA of 256 threads works on the block in global memory (it is L2-resident: 512 KB); per 32-column sub-step:
//   warp 0           : potf2 of the 32 x 32 block, lane = row, the row lives in registers, pivots / multipliers travel
//                      by shuffle (no barrier inside the 32-pivot chain)
//   threads 0..223   : one panel row each (rows below the sub-block inside the diagonal block): x <- x L_ss^-T
//   last warp        : Z = L_ss^-1 (lane = column), needed by chol_trsm_kernel
//   all warps        : rank-32 update of the rest of the diagonal block on the fp64 tensor cores, one 32 x 32 tile
//                      per warp and turn (DMMA: 8 shared-memory loads per 16 MMAs; a scalar FMA loop was bound by
//                      its shared-memory loads)
// Shared-memory row pitch 36 doubles: conflict-free for the DMMA fragment pattern [row g][column tg].
constexpr int DG_LD = LNB + 4;
constexpr int DG_XROWS = LNBO - LNB;          // 224 panel rows at most inside the diagonal block
constexpr int DG_SMEM_DOUBLES = (3 * LNB + DG_XROWS) * DG_LD + LNB;
static_assert(DG_LD == TP, "tile primitives of ba_chol_potf2.cuh use a pitch of 36 doubles");
constexpr int DG_THREADS = 256;    // 255 registers per thread: the register-resident 32-wide rows need them
__global__ void __launch_bounds__(DG_THREADS, 1) chol_diag_kernel(double *A, double *Lout, int ld, int n, int k0, double *linv_all, Scalars *sc)
{
    extern __shared__ __align__(16) double dsm[];
    double (*Ls)[DG_LD] = reinterpret_cast<double (*)[DG_LD]>(dsm);
    double (*Zs)[DG_LD] = reinterpret_cast<double (*)[DG_LD]>(dsm + LNB * DG_LD);
    double (*Ws)[DG_LD] = reinterpret_cast<double (*)[DG_LD]>(dsm + 2 * LNB * DG_LD);
    double (*Xs)[DG_LD] = reinterpret_cast<double (*)[DG_LD]>(dsm + 3 * LNB * DG_LD);
    double *dinv = dsm + (3 * LNB + DG_XROWS) * DG_LD;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;
    const int nb = min(LNBO, n - k0);
    const int nsub = (nb + LNB - 1) / LNB;
    for (int e = tid; e < LNB * DG_LD; e += DG_THREADS) Zs[0][e] = 0.0;       // the strictly upper blocks of Z stay zero
    for (int s = 0; s < nsub; s++) {
        const int c0 = k0 + s * LNB;                      // first matrix column of the sub-block
        const int w = min(LNB, k0 + nb - c0);             // its width
        const int below = max(0, k0 + nb - (c0 + LNB));   // rows below it inside the diagonal block
        const int nblk = (below + LNB - 1) / LNB;
        for (int e = tid; e < LNB * LNB; e += DG_THREADS) {
            const int r = e >> 5, c = e & 31;
            Ls[r][c] = (r < w && c <= r) ? A[(size_t) (c0 + r) * ld + (c0 + c)] : ((r == c) ? 1.0 : 0.0);
        }
        for (int e0 = 0; e0 < nblk * LNB * LNB; e0 += DG_THREADS * 8) {      // 8 independent loads per thread in flight
            double v[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int e = e0 + tid + i * DG_THREADS, r = e >> 5, c = e & 31;
                v[i] = (r < below && c < w) ? A[(size_t) (c0 + LNB + r) * ld + (c0 + c)] : 0.0;
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int e = e0 + tid + i * DG_THREADS;
                if (e < nblk * LNB * LNB) Xs[e >> 5][e & 31] = v[i];
            }
        }
        __syncthreads();
        if (warp == 0) {
            // potf2 of the 32 x 32 block (ba_chol_potf2.cuh): lane = row, 8-column register panels, DMMA rank-8 updates
            const bool bad = warp_potf2_32_tc(Ls, dinv, lane, true);
            if (bad && lane == 0) sc->chol_fail = 1;
        } else if (warp == 1) {
            warp_tile_inverse(Ls, dinv, Zs, Ws, lane);          // Z = L_ss^-1 assembled one panel behind warp 0
        }
        __syncthreads();
        // panel rows below the sub-block: X <- X L_ss^-T = X Z^T, 8-row strips on the fp64 tensor cores
        for (int strip = warp; strip * 8 < below; strip += DG_THREADS / 32) warp_rows_times_ZT(Xs, strip * 8, Zs, lane);
        __syncthreads();
        for (int e = tid; e < LNB * LNB; e += DG_THREADS) {
            const int r = e >> 5, c = e & 31;
            if (r < w && c <= r) Lout[(size_t) (c0 + r) * ld + (c0 + c)] = Ls[r][c];
            linv_all[(size_t) (c0 / LNB) * LNB * LNB + e] = (c <= r) ? Zs[r][c] : 0.0;
        }
        for (int e = tid; e < below * LNB; e += DG_THREADS) {
            const int r = e >> 5, c = e & 31;
            if (c < w) Lout[(size_t) (c0 + LNB + r) * ld + (c0 + c)] = Xs[r][c];
        }
        // rank-32 update of the remaining block: tile (bi, bj), bj <= bi, on the fp64 tensor cores
        for (int blk = warp; blk < nblk * (nblk + 1) / 2; blk += DG_THREADS / 32) {
            int bi = 0, rem = blk;
            while (rem > bi) { rem -= bi + 1; bi++; }
            const int bj = rem;
            // the tile's current values are fetched first: the independent loads stay in flight under the MMAs
            double acc[4][4][2], cur[4][4][2];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int gr = bi * LNB + i * 8 + g;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int gc = bj * LNB + j * 8 + 2 * tg;
                    const double *src = A + (size_t) (c0 + LNB + gr) * ld + (c0 + LNB + gc);
                    cur[i][j][0] = (gr < below && gc <= gr) ? src[0] : 0.0;
                    cur[i][j][1] = (gr < below && gc + 1 <= gr) ? src[1] : 0.0;
                    acc[i][j][0] = 0.0; acc[i][j][1] = 0.0;
                }
            }
#pragma unroll
            for (int ks = 0; ks < LNB; ks += 4) {
                double af[4], bf[4];
#pragma unroll
                for (int i = 0; i < 4; i++) af[i] = Xs[bi * LNB + i * 8 + g][ks + tg];
#pragma unroll
                for (int j = 0; j < 4; j++) bf[j] = Xs[bj * LNB + j * 8 + g][ks + tg];
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int gr = bi * LNB + i * 8 + g;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int gc = bj * LNB + j * 8 + 2 * tg;
                    double *dst = A + (size_t) (c0 + LNB + gr) * ld + (c0 + LNB + gc);
                    if (gr < below && gc <= gr) dst[0] = cur[i][j][0] - acc[i][j][0];
                    if (gr < below && gc + 1 <= gr) dst[1] = cur[i][j][1] - acc[i][j][1];
                }
            }
        }
        __syncthreads();
    }
}

// ---- pre-tiled panel image: the operands of the trailing update --------------------------------------------------
// Written by chol_trsm_kernel next to the panel in Lmat: image row q is matrix row k1 + q (the rows
// below the diagonal block, right-hand side row n included), stored as blocks of 128 rows x 32 k, each the exact shared-memory
// image of one operand stage (32 KB): block (q / 128, c / 32) starts at ((q / 128) * 8 + c / 32) * 4096 doubles, whatever the
// matrix pitch.  Inside a block, row r is 16 units of 16 bytes; k = 8 s + 4 h + t (k8 step s, half h, t = k & 3) is element h
// of unit  u = 4 t + (s ^ (t >> 1) ^ 2 (r & 1)).  So one 16-byte load gives a lane both values (t, t + 4) of an m16n8k8
// fragment row, and the XOR spreads the eight lanes of every quarter warp (rows g, g + 1 for even g; t = 0..3) over the
// eight 16-byte bank groups: the fragment loads are free of bank conflicts without padding
// (tests/test_chol_trailing_swizzle.py enumerates them).
constexpr int SY_BT = CHOL_TILE, SY_BK = 32, SY_KCH = LNBO / SY_BK;      // tile, K chunk, chunks per panel
constexpr int SY_BLOCK = SY_BT * SY_BK;                             // doubles per operand stage (32 KB)
constexpr int SY_STAGES = 3;
constexpr int SY_CONSUMERS = 8, SY_THREADS = 32 * (SY_CONSUMERS + 4);      // two consumer warpgroups + the producer's
// Registers: 168 per thread at launch (384 threads, one CTA per SM); the producer warpgroup gives 128 of them back and the
// consumers take them: 4 warps x 40 + 8 warps x 232 = 12 warps x 168
constexpr int SY_PRODUCER_REGS = 40, SY_CONSUMER_REGS = 232;
// The shared list of a launch's nonzero row blocks: 16-bit entries behind two int counts.  A launch with more row blocks
// (n > 16 K) keeps every tile.  The list is kept this short on purpose: the same kernel with 2 KB or 8 KB more shared memory
// (even without the skip) returned wrong factors of dense systems from n ~ 3800 on (H100, cause not found, DESIGN.md §8).
constexpr int SY_MAX_RB = CHOL_MAX_RB;
constexpr size_t SY_SMEM = (size_t) SY_STAGES * 2 * SY_BLOCK * sizeof(double) + 2 * SY_STAGES * 8 + 2 * sizeof(int) + SY_MAX_RB * sizeof(uint16_t);
__device__ __forceinline__ size_t syrk_img_index(int q, int c)
{
    const int r = q & (SY_BT - 1), k = c & (SY_BK - 1), t = k & 3;
    const int u = 4 * t + ((k >> 3) ^ (t >> 1) ^ ((r & 1) << 1));
    return ((size_t) (q / SY_BT) * SY_KCH + c / SY_BK) * SY_BLOCK + r * SY_BK + 2 * u + ((k >> 2) & 1);
}
// doubles of the image of the first panel (the largest); it lives in xinv_ws, which holds ceil(n/256) * 65536 doubles and is
// not used before the factorisation ends: ceil((n - 255) / 128) <= 2 ceil(n / 256), so it always fits
static size_t syrk_img_doubles(int n) { return (size_t) ((n + 1 - LNBO + SY_BT - 1) / SY_BT) * SY_KCH * SY_BLOCK; }

// ---- panel solve: rows below the diagonal block (and the right-hand side row n) ----------------------------------
// X_s = (B_s - sum_{t<s} X_t L_st^T) Z_ss^T for the eight 32-column sub-blocks s, 64 rows per CTA, X kept in shared
// memory, every product on the fp64 tensor cores (DMMA): warp (wr = warp & 3, wc = warp >> 2) owns the 16 x 16 piece
// [16 wr, +16) x [16 wc, +16) of the current 64 x 32 sub-block as 2 x 2 accumulator tiles.
// Source rows: matrix rows of A below the diagonal block (ident == 0), or rows of the 256 x 256 identity (ident == 1:
// the result is L_kk^-T, the inverse the back substitution multiplies with; blockIdx.y = panel).
// ident == 0 also records one flag per CTA: SLAB_NONZERO when a value it wrote is != 0 (NaN included), SLAB_NONFINITE
// when one is NaN or infinite.  A CTA whose source rows are all +-0 skips the solve and writes +0: what the solve returns
// for them whenever the diagonal block factored (finite L_kk and Z).  Its image rows are written too: the trailing update
// reads them when the other 64 rows of their 128-row block are nonzero.
constexpr int SLAB_NONZERO = 1, SLAB_NONFINITE = 2;
constexpr int TR_ROWS = CHOL_SLAB;
constexpr int TR_LDX = LNBO + 4;       // pitch = 4 (mod 16) doubles: conflict-free DMMA fragment loads
constexpr int TR_LDB = LNB + 4;
constexpr int TR_NLB = LNBO / LNB;      // blocks staged per sub-step: L_s0 .. L_s,s-1 and Z_ss
constexpr int TR_SMEM_DOUBLES = TR_ROWS * TR_LDX + TR_NLB * LNB * TR_LDB;
struct TrsmArgs {
    const double *A;        // ident == 0: source rows (matrix, pitch ld)
    double *dst;            // destination rows: dst[(dst_row0 + r) * dst_ld + dst_col0 + c]
    double *img;            // ident == 0, not null: the rows also go to the panel image of the trailing update
    int *flags;             // ident == 0: the panel's zero flags, flags[blockIdx.x] = SLAB_* bits of the rows this CTA wrote
    const double *Lfac;     // factor matrix (the panel's diagonal block is read from it)
    const double *linv_all;
    int ld, dst_ld, nrows, ident;
    int k0, nb;             // ident == 0: the panel.  ident == 1: panel = blockIdx.y * 256
    int n;
};
__global__ void __launch_bounds__(256) chol_trsm_kernel(const TrsmArgs T)
{
    extern __shared__ double dsm[];
    double *Xs = dsm;                                                                     // [64][260]
    double (*Lb)[LNB][TR_LDB] = reinterpret_cast<double (*)[LNB][TR_LDB]>(dsm + TR_ROWS * TR_LDX);               // [8][32][36]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tg = lane & 3;
    const int k0 = T.ident ? (int) blockIdx.y * LNBO : T.k0;
    const int nb = T.ident ? min(LNBO, T.n - k0) : T.nb;
    const int row0 = T.ident ? (int) blockIdx.x * TR_ROWS : k0 + nb + (int) blockIdx.x * TR_ROWS;   // ident: row of the identity block
    const int rcount = T.ident ? max(0, min(TR_ROWS, nb - row0)) : min(TR_ROWS, T.nrows - row0);
    if (rcount <= 0) return;
    const double *Lfac = T.Lfac;
    const int ld = T.ld;
    bool src_nz = false;
    for (int r0 = 0; r0 < TR_ROWS; r0 += 32) {       // thread = column, 32 rows per batch: 32 independent loads in flight
        double v[32];
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const int r = r0 + i, c = tid;
            v[i] = 0.0;
            if (r < rcount && c < nb) v[i] = T.ident ? ((row0 + r == c) ? 1.0 : 0.0) : T.A[(size_t) (row0 + r) * ld + (k0 + c)];
        }
#pragma unroll
        for (int i = 0; i < 32; i++) { Xs[(r0 + i) * TR_LDX + tid] = v[i]; src_nz |= v[i] != 0.0; }
    }
    const bool src_zero = !T.ident && !__syncthreads_or(src_nz);
    const int nsub = src_zero ? 0 : (nb + LNB - 1) / LNB;
    const int wr = warp & 3, wc = warp >> 2;
    const double *xrow0 = Xs + (wr * 16 + g) * TR_LDX, *xrow1 = xrow0 + 8 * TR_LDX;
    double pre[4 * TR_NLB];      // the blocks of the NEXT sub-step, 4 elements of each per thread
    auto trsm_prefetch = [&](int sn) {
        const int wn = min(LNB, nb - sn * LNB);
#pragma unroll
        for (int t = 0; t < TR_NLB; t++) {
            if (t > sn) continue;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int e = tid + 256 * j, c = e >> 5, u = e & 31;
                double v = 0.0;
                if (t < sn) { if (c < wn) v = Lfac[(size_t) (k0 + sn * LNB + c) * ld + (k0 + t * LNB + u)]; }
                else v = T.linv_all[(size_t) (k0 / LNB + sn) * LNB * LNB + e];
                pre[4 * t + j] = v;
            }
        }
    };
    if (nsub > 0) trsm_prefetch(0);
    __syncthreads();
    for (int s = 0; s < nsub; s++) {
        const int w = min(LNB, nb - s * LNB);
        double acc[2][2][2];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const double *src = Xs + (wr * 16 + i * 8 + g) * TR_LDX + s * LNB + wc * 16 + j * 8 + 2 * tg;
                acc[i][j][0] = src[0]; acc[i][j][1] = src[1];
            }
        // staging: the blocks L_s0 .. L_s,s-1 and Z_ss were requested one sub-step ahead (they depend on nothing computed here),
        // so their L2 latency hides under the previous sub-step's MMAs instead of costing up to four round trips per sub-step
        __syncthreads();
#pragma unroll
        for (int t = 0; t < TR_NLB; t++)
            if (t <= s)
#pragma unroll
                for (int j = 0; j < 4; j++) { const int e = tid + 256 * j; Lb[t][e >> 5][e & 31] = pre[4 * t + j]; }
        __syncthreads();
        if (s + 1 < nsub) trsm_prefetch(s + 1);
        for (int t = 0; t < s; t++) {
#pragma unroll
            for (int ks = 0; ks < LNB; ks += 4) {
                const double a0 = -xrow0[t * LNB + ks + tg], a1 = -xrow1[t * LNB + ks + tg];
                const double b0 = Lb[t][wc * 16 + g][ks + tg], b1 = Lb[t][wc * 16 + 8 + g][ks + tg];
                dmma_m8n8k4(acc[0][0][0], acc[0][0][1], a0, b0); dmma_m8n8k4(acc[0][1][0], acc[0][1][1], a0, b1);
                dmma_m8n8k4(acc[1][0][0], acc[1][0][1], a1, b0); dmma_m8n8k4(acc[1][1][0], acc[1][1][1], a1, b1);
            }
        }
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 2; j++) {
                double *dstp = Xs + (wr * 16 + i * 8 + g) * TR_LDX + s * LNB + wc * 16 + j * 8 + 2 * tg;
                dstp[0] = acc[i][j][0]; dstp[1] = acc[i][j][1];
            }
        __syncthreads();
        double out[2][2][2];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 2; j++) { out[i][j][0] = 0.0; out[i][j][1] = 0.0; }
#pragma unroll
        for (int ks = 0; ks < LNB; ks += 4) {      // X_s = Y Z^T (Z lower triangular: Z[c][u] = 0 for u > c)
            const double a0 = xrow0[s * LNB + ks + tg], a1 = xrow1[s * LNB + ks + tg];
            const double b0 = Lb[s][wc * 16 + g][ks + tg], b1 = Lb[s][wc * 16 + 8 + g][ks + tg];
            dmma_m8n8k4(out[0][0][0], out[0][0][1], a0, b0); dmma_m8n8k4(out[0][1][0], out[0][1][1], a0, b1);
            dmma_m8n8k4(out[1][0][0], out[1][0][1], a1, b0); dmma_m8n8k4(out[1][1][0], out[1][1][1], a1, b1);
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 2; i++) {
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int c = wc * 16 + j * 8 + 2 * tg;
                double *dstp = Xs + (wr * 16 + i * 8 + g) * TR_LDX + s * LNB + c;
                dstp[0] = (c < w) ? out[i][j][0] : 0.0;
                dstp[1] = (c + 1 < w) ? out[i][j][1] : 0.0;
            }
        }
    }
    __syncthreads();
    int bits = 0;
    for (int e = tid; e < TR_ROWS * LNBO; e += 256) {
        const int rr = e >> 8, c = e & 255;
        if (rr < rcount && c < nb) {
            if (T.ident) T.dst[((size_t) blockIdx.y * LNBO + row0 + rr) * LNBO + c] = Xs[rr * TR_LDX + c];
            else {
                const double v = src_zero ? 0.0 : Xs[rr * TR_LDX + c];
                bits |= (v != 0.0 ? SLAB_NONZERO : 0) | (isfinite(v) ? 0 : SLAB_NONFINITE);
                T.dst[(size_t) (row0 + rr) * T.dst_ld + (k0 + c)] = v;
                if (T.img) T.img[syrk_img_index((int) blockIdx.x * TR_ROWS + rr, c)] = v;
            }
        }
    }
    if (!T.ident) {
        const int nz = __syncthreads_or(bits & SLAB_NONZERO), nf = __syncthreads_or(bits & SLAB_NONFINITE);
        if (tid == 0) T.flags[blockIdx.x] = (nz ? SLAB_NONZERO : 0) | (nf ? SLAB_NONFINITE : 0);
    }
}

// ---- trailing update on the fp64 tensor cores (DMMA) -----------------------------------------------
// A[r][c] -= sum_{t < 256} L[r][t] L[c][t]  for c in [cb, ce), r in [c, nrows), over the 128 x 128 tiles of the lower
// triangle only.  PERSISTENT: one CTA per SM walks a static list of tiles (column block by column block; CTA b takes tiles
// b, b + grid, ...), with no atomics and no split K, so the result does not depend on the grid.
// ZERO BLOCKS SKIPPED: the reduced camera system couples only cameras that share points, and its factor keeps many
// 128-row panel blocks at exactly +-0 in the early panels.  The prologue lists the launch's row blocks whose two 64-row slabs
// of the panel solve are not both flagged zero, and the tiles are the lower triangle of that list (columns inside
// [cb, ce)).  A skipped tile changes no bit: with one operand all +-0 every product is +-0, the accumulators stay +0, and
// C - (+0) is C (-0 and NaN included).  That needs the other operand finite, so a launch with a non-finite panel value keeps
// every tile, as does one with more row blocks than the list holds.  Once the factor is dense the list is 0, 1, 2, ... and the tiles are those of the dense triangle.
// WARP-SPECIALISED, 384 threads:
//   warp 8      producer (warps 9..11 only hand their registers to the consumers and leave): a K chunk (32) of one operand of one tile is ONE contiguous 32 KB cp.async.bulk out of the pre-tiled
//               panel image (below) into a ring of SY_STAGES (A, B) stages with full / empty mbarriers.  It runs ahead across
//               tiles, so the next tile's first chunks land while the consumers write the previous tile back, and when it
//               starts on a tile it prefetches that tile's output rows into L2 (the consumers read them a tile later).
//   warps 0..7  consumers, 2 (rows) x 4 (cols), warp tile 64 x 32 = 4 x 4 accumulators of mma.sync.m16n8k8.f64, fed by
//               16-byte fragment loads from the stage; inside a chunk the compiler interleaves the loads of the next k8
//               step with the MMAs of the current one (an explicit register double buffer on top of the 128 accumulator
//               registers spilled).
// The arithmetic is that of every earlier version of this update: accumulators start at zero, k ascends in steps of 8 with
// the same k -> lane mapping, and the tile is written back as C - acc, so the factor does not depend on how the operands
// reach the tensor cores.
// D(16x8) += A(16x8) B(8x8); lane = 4 g + t holds A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4], B[t][g], B[t+4][g],
// D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]
__device__ __forceinline__ void dmma_m16n8k8(double (&d)[4], const double (&a)[4], const double (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

struct SyrkArgs {
    double *A;              // the matrix being factored (pitch ld, nrows rows)
    const double *img;      // panel image; its row 0 is matrix row img_row0
    const int *flags;       // the panel solve's flags, one per 64 image rows (nslab of them)
    int ld, nrows, cb, ce, img_row0, nslab;
    int nrb, ncb;           // row blocks of 128 from cb; column blocks of 128 in [cb, ce)
};

__global__ void __launch_bounds__(SY_THREADS, 1) chol_syrk_dmma_kernel(const SyrkArgs S)
{
    using namespace bsfm::ptx;
    extern __shared__ __align__(128) double ssm[];
    const uint32_t sbase = smem_u32(ssm);
    const uint32_t bar_full = sbase + (uint32_t) (SY_STAGES * 2 * SY_BLOCK * sizeof(double)), bar_empty = bar_full + 8 * SY_STAGES;
    int *counts = reinterpret_cast<int *>(ssm + SY_STAGES * 2 * SY_BLOCK + 2 * SY_STAGES);      // kept row blocks, kept column blocks
    uint16_t *list = reinterpret_cast<uint16_t *>(counts + 2);                                  // [SY_MAX_RB]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < SY_STAGES; s++) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, SY_CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == 0) {      // the row blocks with a nonzero panel block, ascending; how many of them are column blocks
        int nk = S.nrb, nkc = S.ncb;      // every row block: more than the list holds, or a non-finite panel value
        if (S.nrb <= SY_MAX_RB) {
            const int rb0 = (S.cb - S.img_row0) / SY_BT;
            int k = 0, kc = 0;
            bool nonfinite = false;
            for (int r0 = 0; r0 < S.nrb; r0 += 32) {
                const int rb = r0 + lane, s = 2 * (rb0 + rb);
                const int f = (rb < S.nrb) ? S.flags[s] | ((s + 1 < S.nslab) ? S.flags[s + 1] : 0) : 0;
                nonfinite |= __any_sync(0xffffffffu, f & SLAB_NONFINITE);
                const uint32_t m = __ballot_sync(0xffffffffu, f != 0);
                if (f) list[k + __popc(m & ((1u << lane) - 1))] = rb;
                k += __popc(m);
                kc += __popc(m & __ballot_sync(0xffffffffu, rb < S.ncb));
            }
            if (!nonfinite) { nk = k; nkc = kc; }
        }
        if (lane == 0) { counts[0] = nk; counts[1] = nkc; }
    }
    __syncthreads();
    const int nk = counts[0], nkc = counts[1];
    const bool all = nk == S.nrb;      // every row block kept: the list is 0, 1, 2, ... (or was not built)
    const int ntiles = nkc * nk - nkc * (nkc - 1) / 2;
    if ((int) blockIdx.x >= ntiles) return;      // no tile for this CTA: no mbarrier is ever waited on
    const bool vec2 = (S.ld & 1) == 0;      // 16-byte accesses to the output need an even pitch
    // tile t of the launch -> (row block, column block), column block by column block over the lower triangle of the list
    auto tile_of = [&](int t, int &rb, int &cbk) {
        int c = 0;
        while (t >= nk - c) { t -= nk - c; c++; }
        cbk = all ? c : list[c]; rb = all ? c + t : list[c + t];
    };

    if (warp >= SY_CONSUMERS) {
        // ===================== producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(SY_PRODUCER_REGS));
        if (warp != SY_CONSUMERS) return;
        uint64_t keep;      // the panel image is read by a whole column of tiles: keep it in L2
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
        uint32_t st = 0, ph = 0;
        for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
            int rb, cbk;
            tile_of(t, rb, cbk);
            const int r0 = S.cb + rb * SY_BT, c0 = S.cb + cbk * SY_BT;
            const int bytes = (min(SY_BT, S.ce - c0) * 8) & ~15;
            if (vec2 && bytes > 0)
                for (int i = lane; i < SY_BT && r0 + i < S.nrows; i += 32) bulk_prefetch_l2(S.A + (size_t) (r0 + i) * S.ld + c0, bytes);
            if (lane == 0) {
                const double *ga = S.img + (size_t) ((r0 - S.img_row0) / SY_BT) * SY_KCH * SY_BLOCK;
                const double *gb = S.img + (size_t) ((c0 - S.img_row0) / SY_BT) * SY_KCH * SY_BLOCK;
                for (int kc = 0; kc < SY_KCH; kc++) {
                    mbar_wait_backoff(bar_empty + 8 * st, ph ^ 1);
                    mbar_expect_tx(bar_full + 8 * st, 2 * SY_BLOCK * sizeof(double));
                    const uint32_t dst = sbase + st * (uint32_t) (2 * SY_BLOCK * sizeof(double));
                    tma_bulk_g2s_hint(dst, ga + kc * SY_BLOCK, SY_BLOCK * sizeof(double), bar_full + 8 * st, keep);
                    tma_bulk_g2s_hint(dst + SY_BLOCK * sizeof(double), gb + kc * SY_BLOCK, SY_BLOCK * sizeof(double), bar_full + 8 * st, keep);
                    if (++st == SY_STAGES) { st = 0; ph ^= 1; }
                }
            }
            __syncwarp();
        }
        return;
    }

    // ===================== consumers =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(SY_CONSUMER_REGS));
    const int wr = warp >> 2, wc = warp & 3;           // warp tile origin: rows wr*64, cols wc*32
    const int g = lane >> 2, tg = lane & 3;
    // this lane's unit of k8 step s in its rows is 4 tg + (s ^ swz); every fragment row differs from row g by a multiple of 8
    const int swz = (tg >> 1) ^ ((g & 1) << 1);
    const double *lane_a = ssm + (wr * 64 + g) * SY_BK + 8 * tg;
    const double *lane_b = ssm + SY_BLOCK + (wc * 32 + g) * SY_BK + 8 * tg;
    auto load_frags = [&](double (&af)[4][4], double (&bf)[4][2], uint32_t stage, int s) {
        const int off = (int) stage * 2 * SY_BLOCK + 2 * (s ^ swz);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const double2 lo = *reinterpret_cast<const double2 *>(lane_a + off + (i * 16) * SY_BK);
            const double2 hi = *reinterpret_cast<const double2 *>(lane_a + off + (i * 16 + 8) * SY_BK);
            af[i][0] = lo.x; af[i][1] = hi.x; af[i][2] = lo.y; af[i][3] = hi.y;
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const double2 v = *reinterpret_cast<const double2 *>(lane_b + off + (j * 8) * SY_BK);
            bf[j][0] = v.x; bf[j][1] = v.y;
        }
    };
    uint32_t st = 0, ph = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        double acc[4][4][4];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int e = 0; e < 4; e++) acc[i][j][e] = 0.0;
        for (int kc = 0; kc < SY_KCH; kc++) {
            mbar_wait(bar_full + 8 * st, ph);
#pragma unroll
            for (int s = 0; s < 4; s++) {
                double fa[4][4], fb[4][2];
                load_frags(fa, fb, st, s);
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) dmma_m16n8k8(acc[i][j], fa[i], fb[j]);
            }
            __syncwarp();      // the stage's operands are in registers: hand it back to the producer
            if (lane == 0) mbar_arrive(bar_empty + 8 * st);
            if (++st == SY_STAGES) { st = 0; ph ^= 1; }
        }
        int rb, cbk;
        tile_of(t, rb, cbk);
        const int r0 = S.cb + rb * SY_BT, c0 = S.cb + cbk * SY_BT;
        // C - acc in four quarters of 16 rows per warp: every load of a quarter is issued before its first store (the compiler
        // cannot move a load of the matrix past a store to it, so element pair by pair the write-back was 32 serial L2 round
        // trips; halves instead of quarters spill)
#pragma unroll
        for (int h = 0; h < 4; h++) {
            double2 cur[2][4];
#pragma unroll
            for (int pass = 0; pass < 2; pass++) {
#pragma unroll
                for (int ii = 0; ii < 2; ii++) {
                    const int i = 2 * h + ii, r = r0 + wr * 64 + i * 8 + g;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int c = c0 + wc * 32 + j * 8 + 2 * tg;
                        const bool in0 = r < S.nrows && c < S.ce && c <= r;
                        const bool in1 = r < S.nrows && c + 1 < S.ce && c + 1 <= r;      // implies in0
                        double *dst = S.A + (size_t) r * S.ld + c;
                        if (pass == 0) {      // output read once and written once: stream it through L2
                            cur[ii][j] = make_double2(0.0, 0.0);
                            if (vec2 && in1) cur[ii][j] = __ldcs(reinterpret_cast<const double2 *>(dst));
                            else { if (in0) cur[ii][j].x = dst[0]; if (in1) cur[ii][j].y = dst[1]; }
                        } else {
                            const double v0 = cur[ii][j].x - acc[i >> 1][j][2 * (i & 1)], v1 = cur[ii][j].y - acc[i >> 1][j][2 * (i & 1) + 1];
                            if (vec2 && in1) __stcs(reinterpret_cast<double2 *>(dst), make_double2(v0, v1));
                            else { if (in0) dst[0] = v0; if (in1) dst[1] = v1; }
                        }
                    }
                }
            }
        }
    }
}

// A[r][c] -= L[r][k0 : k0 + 256] . L[c][k0 : k0 + 256] over the lower triangle of rows [cb, nrows) x columns [cb, ce), with
// the panel read from its image (row 0 = matrix row img_row0 = k0 + 256) and its flags; at most max_ctas persistent CTAs.
// The grid is that of the dense triangle: how many tiles are kept is known only on the device.
static void syrk_dmma(cudaStream_t st, double *A, const double *img, const int *flags, int nslab, int ld, int nrows, int cb, int ce,
                      int img_row0, int max_ctas)
{
    SyrkArgs S = {};
    S.A = A; S.img = img; S.flags = flags; S.nslab = nslab; S.ld = ld; S.nrows = nrows; S.cb = cb; S.ce = ce; S.img_row0 = img_row0;
    S.nrb = (nrows - cb + SY_BT - 1) / SY_BT;
    S.ncb = (ce - cb + SY_BT - 1) / SY_BT;      // <= nrb: ce <= n < nrows
    const int ntiles = S.ncb * S.nrb - S.ncb * (S.ncb - 1) / 2;
    chol_syrk_dmma_kernel<<<std::min(ntiles, max_ctas), SY_THREADS, SY_SMEM, st>>>(S);
}

// The lower-triangle elements (right-hand-side row included) of the tiles chol_syrk_dmma_kernel keeps in that launch, from
// the panel's flags read back to the host: the trailing update's executed FLOPs are 2 x 256 x this
static double syrk_kept_elements(const int *flags, int nslab, int nrows, int cb, int ce, int img_row0)
{
    const int nrb = (nrows - cb + SY_BT - 1) / SY_BT, ncb = (ce - cb + SY_BT - 1) / SY_BT, rb0 = (cb - img_row0) / SY_BT;
    std::vector<int> list;
    bool nonfinite = false;
    for (int rb = 0; rb < nrb; rb++) {
        const int s = 2 * (rb0 + rb), f = flags[s] | ((s + 1 < nslab) ? flags[s + 1] : 0);
        nonfinite |= (f & SLAB_NONFINITE) != 0;
        if (f) list.push_back(rb);
    }
    if (nonfinite || nrb > SY_MAX_RB) { list.resize(nrb); for (int rb = 0; rb < nrb; rb++) list[rb] = rb; }
    double el = 0.0;
    for (size_t j = 0; j < list.size() && list[j] < ncb; j++) {
        const int c0 = cb + list[j] * SY_BT, c1 = std::min(c0 + SY_BT, ce);
        for (size_t i = j; i < list.size(); i++) {
            const int r0 = cb + list[i] * SY_BT, r1 = std::min(r0 + SY_BT, nrows);
            for (int c = c0; c < c1; c++) el += std::max(0, r1 - std::max(r0, c));
        }
    }
    return el;
}

// ---- back substitution L^T x = y, one launch per outer panel (last to first) --------------------------------------
// y lives in row n of the factor matrix and is updated in place.  Every CTA first forms the panel's own 256 unknowns
// x_p = L_pp^-T y_p with the inverse computed after the factorisation (Xinv = L_pp^-T, row-major 256 x 256, upper
// triangular; one warp per row, coalesced), then CTA b removes their contribution from 64 of the remaining right-hand
// side entries:  y[c] -= sum_r L[k0 + r][c] x[r].
__global__ void __launch_bounds__(1024) chol_backsolve_big_kernel(double *L, int ld, int n, int k0, int nb, const double *Xinv_all, double *x)
{
    __shared__ double ys[LNBO];
    __shared__ double xs[LNBO];
    __shared__ double part[16][64];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double *y = L + (size_t) n * ld;
    if (tid < LNBO) ys[tid] = (tid < nb) ? y[k0 + tid] : 0.0;
    __syncthreads();
    const double *Xi = Xinv_all + (size_t) (k0 / LNBO) * LNBO * LNBO;
    {   // warp = 8 rows of x_p; all 64 loads of a lane are independent (one memory round trip)
        const int i0 = warp * 8;
        double a[8];
#pragma unroll
        for (int u = 0; u < 8; u++) a[u] = 0.0;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int c = lane + 32 * q;
            const double yv = ys[c];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i = i0 + u;
                const double zv = (c >= i && c < nb && i < nb) ? Xi[(size_t) i * LNBO + c] : 0.0;
                a[u] = fma(zv, yv, a[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) a[u] += shfl_d(a[u], lane ^ o);
            if (lane == 0) { xs[i0 + u] = a[u]; if (blockIdx.x == 0 && i0 + u < nb) x[k0 + i0 + u] = a[u]; }
        }
    }
    __syncthreads();
    const int col = blockIdx.x * 64 + (tid & 63), grp = tid >> 6;      // 16 row groups of 16
    double acc = 0.0;
    if (col < k0) {
        const int r_lo = grp * 16;
#pragma unroll
        for (int q = 0; q < 16; q++) {
            const int rr = r_lo + q;
            if (rr < nb) acc = fma(L[(size_t) (k0 + rr) * ld + col], xs[rr], acc);
        }
    }
    part[grp][tid & 63] = acc;
    __syncthreads();
    if (tid < 64 && col < k0) {
        double sacc = 0.0;
#pragma unroll
        for (int q = 0; q < 16; q++) sacc += part[q][tid];
        y[col] -= sacc;
    }
}


// ---- optional per-kernel-class device timing (bench.py's roofline of the dominant kernel; off by default) --------
namespace {
struct CholProfile {
    bool on = false;
    float ms[4] = {0, 0, 0, 0};          // diag, trsm, trailing update, back substitution
    int launches[4] = {0, 0, 0, 0};
    double fp64_flops = 0.0;      // trailing update only, the tiles it executed
    struct Update { size_t flag_off; int nslab, cb, ce, img_row0; };
    std::vector<Update> updates;  // the trailing-update launches of the factorisation in flight
    std::vector<cudaEvent_t> pool;
    size_t used = 0;
    struct Span { int cls; cudaEvent_t a, b; };
    std::vector<Span> spans;
    std::vector<size_t> open;     // spans begun and not yet ended, innermost last (the look-ahead's diagonal block nests in an update)
    cudaEvent_t get() { if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); } return pool[used++]; }
    void begin(int cls, cudaStream_t st) { if (!on) return; Span sp{cls, get(), get()}; cudaEventRecord(sp.a, st); open.push_back(spans.size()); spans.push_back(sp); }
    void end(cudaStream_t st) { if (!on) return; const Span &sp = spans[open.back()]; open.pop_back(); cudaEventRecord(sp.b, st); launches[sp.cls]++; }
    void collect()
    {
        for (auto &sp : spans) { cudaEventSynchronize(sp.b); float t = 0; cudaEventElapsedTime(&t, sp.a, sp.b); ms[sp.cls] += t; }
        spans.clear(); open.clear(); used = 0;
    }
};
thread_local CholProfile g_prof;
}  // namespace

static int set_smem_attr_once(int dev)
{
    static std::atomic<int> done[64];
    if (dev < 0 || dev >= 64) return BSFM_OK;
    if (done[dev].load(std::memory_order_acquire)) return BSFM_OK;
    BSFM_CUDA_TRY(cudaFuncSetAttribute(chol_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) (DG_SMEM_DOUBLES * sizeof(double))));
    BSFM_CUDA_TRY(cudaFuncSetAttribute(chol_trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) (TR_SMEM_DOUBLES * sizeof(double))));
    BSFM_CUDA_TRY(cudaFuncSetAttribute(chol_syrk_dmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) SY_SMEM));
    done[dev].store(1, std::memory_order_release);
    return BSFM_OK;
}

// Same contract as chol_solve (ba_chol.cu): symmetric A (both triangles) + right-hand side in row n; Lmat (n+1) x n;
// linv_ws ceil(n/32) * 1024 doubles; xinv_ws ceil(n/256) * 65536 doubles (L_pp^-T of every panel); x receives the solution.
// band: a fitting envelope plan (ba_order.cu: chol_band_plan).  The system then takes the one-launch band factorisation and the
// envelope-bounded back substitution instead of the panels below (entries of A outside the envelope are taken as zero).
int chol_solve_large(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *xinv_ws, double *x, Scalars *sc,
                     const CholBand *band)
{
    if (band && band->env) {
        g_prof.begin(0, st);
        int rc = chol_band_factor(st, A, Lmat, n, linv_ws, *band, sc);
        g_prof.end(st);
        if (rc != BSFM_OK) return rc;
        g_prof.begin(3, st);
        rc = chol_band_backsolve(st, Lmat, n, linv_ws, *band, x);
        g_prof.end(st);
        return rc;
    }
    const int ld = n, nrows = n + 1;
    int dev = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    { int rc = set_smem_attr_once(dev); if (rc != BSFM_OK) return rc; }
    int sms = 0;
    BSFM_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // the trailing update reads each panel from its pre-tiled image, kept in xinv_ws until the panel inverses need it
    double *img = xinv_ws;
    if (syrk_img_doubles(n) > (size_t) ((n + LNBO - 1) / LNBO) * LNBO * LNBO || (reinterpret_cast<uintptr_t>(img) & 15) != 0) {
        set_error("chol_solve_large: the panel image does not fit the 16-byte aligned xinv workspace");
        return BSFM_ERR_ARG;
    }
    // the zero flags of every panel solve (a stride of one flag per 64 rows of the whole matrix per panel) at the end of linv_ws
    int *flags = reinterpret_cast<int *>(linv_ws + chol_large_flags_offset(n));
    const size_t flag_stride = (size_t) (nrows + TR_ROWS - 1) / TR_ROWS;
    if (chol_large_flags_offset(n) + (chol_large_flag_count(n) + 1) / 2 > chol_ws_doubles(n) ||
        (size_t) ((n + LNBO - 1) / LNBO) * flag_stride > chol_large_flag_count(n)) {
        set_error("chol_solve_large: the zero flags of n = %d do not fit the workspace", n);
        return BSFM_ERR_ARG;
    }
    // Look-ahead: the diagonal block of panel p+1 is a serial chain on ONE SM.  The trailing update of panel p is therefore
    // split into the tile columns panel p+1 lives in (launched first) and the rest, and diag(p+1) runs on a side stream next
    // to the rest, taking the first SM the rest's CTAs leave free:
    //   main : trsm(p)  col(p) -E1->  rest(p) ............ -wait E2->  trsm(p+1) ...
    //   side :                 wait E1  diag(p+1) -E2->
    // The update's CTAs are persistent and hold their SMs to the end, so the rest runs on one SM fewer than the GPU has: that
    // SM is diag(p+1)'s.
    // BSFM_BA_CHOL_LOOKAHEAD=0 serialises everything on the main stream.
    static const bool lookahead = []() { const char *e = getenv("BSFM_BA_CHOL_LOOKAHEAD"); return !(e && e[0] == '0'); }();
    struct SideStream { int device = -1; cudaStream_t st = nullptr; cudaEvent_t e_col = nullptr, e_diag = nullptr; };
    static thread_local SideStream side;
    if (lookahead && side.device != dev) {
        if (side.st) { cudaStreamDestroy(side.st); cudaEventDestroy(side.e_col); cudaEventDestroy(side.e_diag); side = SideStream(); }
        BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&side.st, cudaStreamNonBlocking));
        BSFM_CUDA_TRY(cudaEventCreateWithFlags(&side.e_col, cudaEventDisableTiming));
        BSFM_CUDA_TRY(cudaEventCreateWithFlags(&side.e_diag, cudaEventDisableTiming));
        side.device = dev;
    }
    bool diag_done = false;       // diag(p) already issued by the look-ahead of panel p-1
    // The last panels are latency-bound (a serial diagonal chain per panel that no trailing update hides any more): once the
    // remaining matrix fits the one-launch dataflow factorisation (ba_chol_dataflow.cu, <= 640), it takes over in place -- same
    // factor blocks, same 32 x 32 inverses, so the batched panel inverses and the back substitution below do not notice.
    static const int tail_max = []() { const char *e = getenv("BSFM_BA_CHOL_TAIL"); return e ? atoi(e) : CHOL_TAIL_MAX; }();
    auto tail_fits = [&](int kk) { return kk > 0 && kk < n && n - kk <= tail_max && n - kk > 2 * LNB; };
    for (int k0 = 0; k0 < n; k0 += LNBO) {
        const int nb = std::min(LNBO, n - k0);
        const int k1 = k0 + nb;
        if (!diag_done && tail_fits(k0)) {
            bool used = false;
            g_prof.begin(0, st);
            int rc = chol_dataflow_factor(st, A + (size_t) k0 * ld + k0, Lmat + (size_t) k0 * ld + k0, ld, n - k0, linv_ws + (size_t) (k0 / LNB) * LNB * LNB,
                                          linv_ws + chol_large_pub_offset(n), sc, &used);
            g_prof.end(st);
            if (rc != BSFM_OK) return rc;
            if (used) break;
        }
        if (!diag_done) {
            g_prof.begin(0, st);
            chol_diag_kernel<<<1, DG_THREADS, DG_SMEM_DOUBLES * sizeof(double), st>>>(A, Lmat, ld, n, k0, linv_ws, sc);
            BSFM_KERNEL_CHECK();
            g_prof.end(st);
        } else {
            BSFM_CUDA_TRY(cudaStreamWaitEvent(st, side.e_diag, 0));
        }
        diag_done = false;
        const int rows_below = nrows - k1;     // >= 1: the right-hand side row
        g_prof.begin(1, st);
        const int nslab = (rows_below + TR_ROWS - 1) / TR_ROWS;
        const size_t flag_off = (size_t) (k0 / LNBO) * flag_stride;      // one flag array per panel: still readable after the factorisation
        TrsmArgs T = {};
        T.A = A; T.dst = Lmat; T.Lfac = Lmat; T.linv_all = linv_ws; T.ld = ld; T.dst_ld = ld; T.nrows = nrows; T.ident = 0; T.k0 = k0; T.nb = nb; T.n = n;
        T.img = (k1 < n) ? img : nullptr;      // k1 < n: a full 256-column panel with a trailing update
        T.flags = flags + flag_off;
        chol_trsm_kernel<<<nslab, 256, TR_SMEM_DOUBLES * sizeof(double), st>>>(T);
        BSFM_KERNEL_CHECK();
        g_prof.end(st);
        if (k1 < n) {
            g_prof.begin(2, st);
            auto update = [&](int cb, int ce, int max_ctas) {
                syrk_dmma(st, A, img, flags + flag_off, nslab, ld, nrows, cb, ce, k1, max_ctas);
                if (g_prof.on) g_prof.updates.push_back({flag_off, nslab, cb, ce, k1});
            };
            const int k2 = std::min(n, k1 + LNBO);      // the columns of panel p+1
            if (lookahead && k2 < n && !tail_fits(k1)) {
                update(k1, k2, sms);
                BSFM_KERNEL_CHECK();
                BSFM_CUDA_TRY(cudaEventRecord(side.e_col, st));
                BSFM_CUDA_TRY(cudaStreamWaitEvent(side.st, side.e_col, 0));
                g_prof.begin(0, side.st);
                chol_diag_kernel<<<1, DG_THREADS, DG_SMEM_DOUBLES * sizeof(double), side.st>>>(A, Lmat, ld, n, k1, linv_ws, sc);
                BSFM_KERNEL_CHECK();
                g_prof.end(side.st);
                BSFM_CUDA_TRY(cudaEventRecord(side.e_diag, side.st));
                diag_done = true;
                update(k2, n, sms - 1);
            } else {
                update(k1, n, sms);
            }
            BSFM_KERNEL_CHECK();
            g_prof.end(st);
        }
    }
    if (diag_done) BSFM_CUDA_TRY(cudaStreamWaitEvent(st, side.e_diag, 0));
    g_prof.begin(3, st);
    // L_pp^-T of every panel at once (the panel solve applied to the rows of the identity), then the back substitution
    const int npan = (n + LNBO - 1) / LNBO;
    double *xinv = xinv_ws;
    {
        TrsmArgs T = {};
        T.A = nullptr; T.dst = xinv; T.Lfac = Lmat; T.linv_all = linv_ws; T.ld = ld; T.dst_ld = LNBO; T.nrows = 0; T.ident = 1; T.k0 = 0; T.nb = 0; T.n = n;
        chol_trsm_kernel<<<dim3(LNBO / TR_ROWS, npan), 256, TR_SMEM_DOUBLES * sizeof(double), st>>>(T);
        BSFM_KERNEL_CHECK();
    }
    for (int k0 = (npan - 1) * LNBO; k0 >= 0; k0 -= LNBO) {
        const int nb = std::min(LNBO, n - k0);
        chol_backsolve_big_kernel<<<std::max(1, (k0 + 63) / 64), 1024, 0, st>>>(Lmat, ld, n, k0, nb, xinv, x);
        BSFM_KERNEL_CHECK();
    }
    g_prof.end(st);
    if (g_prof.on) {
        g_prof.launches[3] += npan;     // end() counted one
        // the FLOPs of the tiles the trailing update executed: the flags are read back before the next factorisation reuses them
        std::vector<int> hflags(chol_large_flag_count(n));
        BSFM_CUDA_TRY(cudaMemcpyAsync(hflags.data(), flags, hflags.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));
        for (const auto &u : g_prof.updates)
            g_prof.fp64_flops += 2.0 * LNBO * syrk_kept_elements(hflags.data() + u.flag_off, u.nslab, nrows, u.cb, u.ce, u.img_row0);
        g_prof.updates.clear();
    }
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm

extern "C" int bsfm_ba_chol_profile(int enable)
{
    using namespace bsfm::ba;
    g_prof.collect();
    for (int q = 0; q < 4; q++) { g_prof.ms[q] = 0; g_prof.launches[q] = 0; }
    g_prof.fp64_flops = 0.0;
    g_prof.updates.clear();
    g_prof.on = enable != 0;
    return BSFM_OK;
}
extern "C" int bsfm_ba_chol_profile_read(float ms[4], int launches[4], double *fp64_flops)
{
    using namespace bsfm::ba;
    g_prof.collect();
    for (int q = 0; q < 4; q++) { if (ms) ms[q] = g_prof.ms[q]; if (launches) launches[q] = g_prof.launches[q]; }
    if (fp64_flops) *fp64_flops = g_prof.fp64_flops;
    return BSFM_OK;
}
