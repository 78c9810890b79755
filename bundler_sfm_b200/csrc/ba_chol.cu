// ba_chol.cu -- dense SPD solve of the reduced camera system S da = E (SURVEY.md K6).
// Reference: sba_Axb_Chol = LAPACK dpotrf + dpotrs, lib/sba-1.5/sba_lapack.c:374-485.
//
// fp64 blocked right-looking Cholesky (lower, row-major, factor written OUT OF PLACE to Lmat) with the
// right-hand side carried as an extra matrix row (row n), so the forward substitution L y = E falls out
// of the factorisation.
//
//   per 32-column step : chol_step_kernel  ONE launch; every CTA redundantly factors the 32x32 diagonal
//                        block fused with the row solves of the two panel blocks its 32x32 trailing tile
//                        needs (16 warps, right-looking, one barrier per pivot, rsqrt + multiply on the
//                        pivot chain), then applies the rank-32 update to its tile
//   end                : chol_backsolve_blocked_kernel (1 CTA) L^T x = y with the inverted diagonal blocks
// This file is the dispatcher (chol_solve) and the FUSED-STEP path for systems of 641..1536 (latency-bound by the sequential
// pivots).  Systems <= 640 go to the one-launch dataflow factorisation (ba_chol_dataflow.cu), systems > 1536 to the 256-column
// panel path with the fp64 tensor-core trailing update (ba_chol_large.cu).
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"
#include "common.h"

namespace bsfm {
namespace ba {

int chol_solve_dataflow(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *x, Scalars *sc, bool *used);

constexpr int NB = 32;

// ---- small systems, one launch per 32-column step ---------------------------------------------------
// Every CTA redundantly factors the 32x32 diagonal block (one warp, rows in registers, pivots and
// multipliers exchanged with shuffles), solves the two 32-row panel blocks its tile needs (one warp
// each, row in registers, L_kk broadcast from shared memory) and applies the rank-32 update to its
// 32x32 tile of the trailing matrix.  Redundant panel work costs no latency and removes the separate
// panel / TRSM launches: the critical path per step is potf2 -> trsm -> update inside one kernel.
// Row block index nbk (= one row) is the right-hand side carried along as matrix row n.
// (loops over shared memory, not unrolled register code: a kernel this short must not spend its time
// fetching tens of KB of straight-line instructions)
constexpr int CST = 512;      // threads of chol_step_kernel
constexpr int CSW = CST / 32;
__global__ void __launch_bounds__(CST) chol_step_kernel(double *A, double *Lout, int ld, int n, int k, int cend, double *Linv_all, Scalars *sc)
{
    __shared__ double Lk[NB][NB + 1];
    __shared__ double Xr[NB][NB + 1];
    __shared__ double Xc[NB][NB + 1];
    __shared__ double dinv[NB];
    __shared__ int fail_s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nbk = (n + NB - 1) / NB;           // matrix row blocks; block nbk = RHS row
    const int k0 = k * NB, nb = min(NB, n - k0);
    // programmatic dependent launch: this grid may be scheduled while its predecessor drains; nothing the
    // predecessor wrote is touched before this point
    cudaGridDependencySynchronize();
    // tile of this CTA: blockIdx 0 = panel owner (no tile); else (cb, rb), k < cb <= rb <= nbk, cb < cend <= nbk
    // (cend = k + 1: the diagonal-only launch that precedes chol_tile_kernel)
    int cb = -1, rb = nbk;                        // the owner solves the RHS row segment
    bool writeback = true;
    if (blockIdx.x > 0) {
        int t = blockIdx.x - 1;
        bool found = false;
        for (int c = k + 1; c < cend; c++) {
            const int cnt = nbk - c + 1;
            if (t < cnt) { cb = c; rb = c + t; found = true; break; }
            t -= cnt;
        }
        // first-column tiles write their panel row block back; when no column is left (k + 1 == cend)
        // dedicated panel-only CTAs do it for the row blocks below
        if (found) writeback = (cb == k + 1); else rb = k + 1 + t;
    }
    const int crow0 = cb * NB;
    const int rrows = (rb == nbk) ? 1 : min(NB, n - rb * NB);        // valid rows in the rb block
    const int rbase = (rb == nbk) ? n : rb * NB;                      // first matrix row of the rb block
    const int crows = (cb >= 0) ? min(NB, n - crow0) : 0;
    // the owner CTA runs the identity through the second row-solve slot: I L_kk^-T = (L_kk^-1)^T comes out of the
    // fused loop for free (needed by the blocked back substitution and by chol_tile_kernel)
    const bool owner = blockIdx.x == 0;
    const bool need_c = owner || (cb >= 0 && cb != rb);

    if (tid == 0) fail_s = 0;
    for (int e = tid; e < NB * NB; e += CST) {
        const int r = e >> 5, c = e & 31;
        Lk[r][c] = (r < nb && c <= r) ? A[(size_t) (k0 + r) * ld + (k0 + c)] : ((r == c) ? 1.0 : 0.0);
        Xr[r][c] = (r < rrows && c < nb) ? A[(size_t) (rbase + r) * ld + (k0 + c)] : 0.0;
        if (owner) Xc[r][c] = (r == c) ? 1.0 : 0.0;
        else if (need_c) Xc[r][c] = (r < crows && c < nb) ? A[(size_t) (crow0 + r) * ld + (k0 + c)] : 0.0;
    }
    __syncthreads();
    // potf2 of L_kk fused with the row solves X <- X L_kk^-T, right-looking, all 8 warps:
    //   thread (lane r, warp g) owns rows r and columns c = g, g+8, g+16, g+24.
    //   Every warp recomputes the pivot reciprocal and the multipliers l_r = a_rj / sqrt(d) of column j
    //   in registers (no communication), updates its own columns of L_kk, Xr and Xc, one barrier per pivot.
    //   Column j itself is left un-scaled in shared memory (it is read-only from now on) and rescaled by
    //   dinv[j] after the loop.  The pivot chain is the latency floor of the whole solve: rsqrt + multiply
    //   instead of sqrt + divide.
    for (int j = 0; j < nb; j++) {
        const double d = Lk[j][j];
        const double arj = Lk[lane][j];
        const double xr = Xr[lane][j];
        const double xc = need_c ? Xc[lane][j] : 0.0;
        const bool bad = !(d > 0.0) || !isfinite(d);
        const double rinv = bad ? 1.0 : rsqrt(d);
        const double l = (lane > j) ? arj * rinv : 0.0;
        const double xjr = xr * rinv, xjc = xc * rinv;
        if (tid == 0) { dinv[j] = rinv; if (bad) fail_s = 1; }
#pragma unroll
        for (int q = 0; q < NB / CSW; q++) {
            const int c = warp + CSW * q;                    // warp-uniform
            if (c > j && c < nb) {
                const double lc = __shfl_sync(0xffffffffu, l, c);   // L[c][j]
                if (lane >= c) Lk[lane][c] = fma(-l, lc, Lk[lane][c]);
                Xr[lane][c] = fma(-xjr, lc, Xr[lane][c]);
                if (need_c) Xc[lane][c] = fma(-xjc, lc, Xc[lane][c]);
            }
        }
        __syncthreads();
    }
    if (tid < NB && tid >= nb) dinv[tid] = 1.0;
    __syncthreads();
    // rescale: L[r][c] = a_rc dinv[c] (c < r), L[c][c] = d_c dinv[c], X[r][c] *= dinv[c]
    for (int e = tid; e < NB * NB; e += CST) {
        const int r = e >> 5, c = e & 31;
        const double sc_c = dinv[c];
        if (c <= r && r < nb) Lk[r][c] *= sc_c;
        Xr[r][c] *= sc_c;
        if (need_c) Xc[r][c] *= sc_c;
    }
    __syncthreads();
    if (warp == 4 && owner) {
        for (int c = 0; c < nb; c++) if (lane < nb && c <= lane) Lout[(size_t) (k0 + lane) * ld + (k0 + c)] = Lk[lane][c];
        if (lane == 0 && fail_s) sc->chol_fail = 1;
    }
    __syncthreads();
    if (owner) {   // Z = L_kk^-1 = Xc^T (lower triangular)
        for (int e = tid; e < NB * NB; e += CST) { const int r = e >> 5, c = e & 31; Linv_all[(size_t) k * NB * NB + e] = (c <= r) ? Xc[c][r] : 0.0; }
    }
    // panel write-back goes to the SEPARATE factor matrix Lout: other CTAs of this launch (possibly in a later
    // wave) still read the un-solved panel blocks from A, so A's panel columns must not change during the step.
    // The owner writes the RHS segment, first-column tiles write their row block
    if (writeback) {
        for (int e = tid; e < NB * NB; e += CST) {
            const int r = e >> 5, c = e & 31;
            if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
        }
    }
    if (cb < 0) return;
    // trailing tile (rb, cb):  A[r][c] -= sum_t Xr[r][t] Xc[c][t]   (c <= r on the diagonal tile)
    const double (*XC)[NB + 1] = need_c ? Xc : Xr;
#pragma unroll
    for (int q = 0; q < NB * NB / CST; q++) {
        const int e = tid + q * CST;
        const int r = e >> 5, c = e & 31;
        if (r < rrows && c < crows && (rb != cb || c <= r)) {
            double acc = 0.0;
#pragma unroll 8
            for (int t = 0; t < NB; t++) acc = fma(Xr[r][t], XC[c][t], acc);
            A[(size_t) (rbase + r) * ld + (crow0 + c)] -= acc;
        }
    }
}

// ---- large grids: tile kernel that takes L_kk^-1 from a preceding diagonal-only chol_step launch -------
// When a step has far more tiles than the GPU holds at once, redoing the 32-pivot chain in every CTA costs
// throughput instead of hiding latency.  The step is then split: chol_step_kernel<<<1>>> factors the diagonal
// block (and solves the RHS segment), and this kernel forms the panel blocks with one small GEMM
// X = B Z^T (Z = L_kk^-1, lower triangular) before the rank-32 tile update.  Same tile enumeration and the
// same out-of-place write-back rules as chol_step_kernel (without its CTA 0).
__global__ void __launch_bounds__(256) chol_tile_kernel(double *A, double *Lout, int ld, int n, int k, int cend, const double *Linv_all)
{
    __shared__ double Zs[NB][NB + 1];
    __shared__ double Br[NB][NB + 1];
    __shared__ double Bc[NB][NB + 1];
    __shared__ double Xr[NB][NB + 1];
    __shared__ double Xc[NB][NB + 1];
    const int tid = threadIdx.x;
    const int nbk = (n + NB - 1) / NB;
    const int k0 = k * NB, nb = min(NB, n - k0);
    int cb = -1, rb = nbk;
    bool writeback = true;
    {
        int t = blockIdx.x;
        bool found = false;
        for (int c = k + 1; c < cend; c++) {
            const int cnt = nbk - c + 1;
            if (t < cnt) { cb = c; rb = c + t; found = true; break; }
            t -= cnt;
        }
        if (found) writeback = (cb == k + 1); else rb = k + 1 + t;
    }
    const int crow0 = cb * NB;
    const int rrows = (rb == nbk) ? 1 : min(NB, n - rb * NB);
    const int rbase = (rb == nbk) ? n : rb * NB;
    const int crows = (cb >= 0) ? min(NB, n - crow0) : 0;
    const bool need_c = cb >= 0 && cb != rb;
    const double *Z = Linv_all + (size_t) k * NB * NB;
    for (int e = tid; e < NB * NB; e += 256) {
        const int r = e >> 5, c = e & 31;
        Zs[r][c] = Z[e];
        Br[r][c] = (r < rrows && c < nb) ? A[(size_t) (rbase + r) * ld + (k0 + c)] : 0.0;
        if (need_c) Bc[r][c] = (r < crows && c < nb) ? A[(size_t) (crow0 + r) * ld + (k0 + c)] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int e = tid + q * 256;
        const int r = e >> 5, c = e & 31;
        double xr = 0.0, xc = 0.0;
        for (int t = 0; t <= c; t++) {
            const double z = Zs[c][t];
            xr = fma(Br[r][t], z, xr);
            if (need_c) xc = fma(Bc[r][t], z, xc);
        }
        Xr[r][c] = xr;
        if (need_c) Xc[r][c] = xc;
    }
    __syncthreads();
    if (writeback) {
        for (int e = tid; e < NB * NB; e += 256) {
            const int r = e >> 5, c = e & 31;
            if (r < rrows && c < nb) Lout[(size_t) (rbase + r) * ld + (k0 + c)] = Xr[r][c];
        }
    }
    if (cb < 0) return;
    const double (*XC)[NB + 1] = need_c ? Xc : Xr;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int e = tid + q * 256;
        const int r = e >> 5, c = e & 31;
        if (r < rrows && c < crows && (rb != cb || c <= r)) {
            double acc = 0.0;
#pragma unroll 8
            for (int t = 0; t < NB; t++) acc = fma(Xr[r][t], XC[c][t], acc);
            A[(size_t) (rbase + r) * ld + (crow0 + c)] -= acc;
        }
    }
}

// ---- back substitution L^T x = y (y = row n of A) with inverted diagonal blocks, single CTA ---------
// per 32-row block (last to first): x_k = L_kk^-T y_k, then y[0:k0] -= L[k0:k0+nb, 0:k0]^T x_k.
// Two barriers per block instead of one per row.
__global__ void __launch_bounds__(512) chol_backsolve_blocked_kernel(const double *A /* factor matrix L, RHS y in row n */, int ld, int n, const double *Linv_all, double *x, double *ywork)
{
    __shared__ double xk[NB];
    __shared__ double ys[NB];
    __shared__ double Li[NB][NB + 1];
    const int tid = threadIdx.x;
    cudaGridDependencySynchronize();
    const double *yrow = A + (size_t) n * ld;
    // y lives in registers for the first 512 columns per thread and in `ywork` (global) beyond that
    double y0 = (tid < n) ? yrow[tid] : 0.0;
    for (int c = tid + 512; c < n; c += 512) ywork[c] = yrow[c];
    const int nbk = (n + NB - 1) / NB;
    // Nothing loaded here depends on x: the inverse block of step kb - 1 is fetched one step ahead and this thread's column of
    // the 32 factor rows of step kb - 1 is requested the moment the registers of step kb are dead, so the L2 latency of both
    // hides under the shared-memory part of the step (the steps are otherwise a chain of dependent global loads).
    double z0 = 0.0, z1 = 0.0, l[NB];
    {
        const int kb = nbk - 1, k0 = kb * NB, nb = min(NB, n - k0);
        z0 = Linv_all[(size_t) kb * NB * NB + tid]; z1 = Linv_all[(size_t) kb * NB * NB + 512 + tid];
#pragma unroll
        for (int r = 0; r < NB; r++) l[r] = (tid < k0 && r < nb) ? A[(size_t) (k0 + r) * ld + tid] : 0.0;
    }
    for (int kb = nbk - 1; kb >= 0; kb--) {
        const int k0 = kb * NB, nb = min(NB, n - k0);
        if (tid >= k0 && tid < k0 + nb) ys[tid - k0] = y0;
        for (int c = tid + 512; c < k0 + nb; c += 512) if (c >= k0) ys[c - k0] = ywork[c];
        Li[tid >> 5][tid & 31] = z0;
        Li[16 + (tid >> 5)][tid & 31] = z1;
        if (kb > 0) { z0 = Linv_all[(size_t) (kb - 1) * NB * NB + tid]; z1 = Linv_all[(size_t) (kb - 1) * NB * NB + 512 + tid]; }
        __syncthreads();
        // x_k = L_kk^-T y_k : 8 lanes per output, 4 terms each, shuffle-reduced
        if (tid < 256) {
            const int o = tid >> 3, part = tid & 7;
            double sacc = 0.0;
#pragma unroll
            for (int u = 0; u < 4; u++) { const int r = part * 4 + u; if (r >= o && r < nb) sacc = fma(Li[r][o], ys[r], sacc); }
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 1);
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 2);
            sacc += __shfl_xor_sync(0xffffffffu, sacc, 4);
            if (part == 0) { xk[o] = sacc; if (o < nb) x[k0 + o] = sacc; }
        }
        __syncthreads();
        {
            double sacc = 0.0;
#pragma unroll
            for (int r = 0; r < NB; r++) sacc = fma(l[r], xk[r], sacc);
            y0 -= sacc;
        }
        for (int c = tid + 512; c < k0; c += 512) {      // systems beyond 512 columns: 16 rows at a time (register budget)
            double sacc = 0.0;
#pragma unroll 1
            for (int r0 = 0; r0 < NB; r0 += 16) {
                double lv[16];
#pragma unroll
                for (int r = 0; r < 16; r++) lv[r] = (r0 + r < nb) ? A[(size_t) (k0 + r0 + r) * ld + c] : 0.0;
#pragma unroll
                for (int r = 0; r < 16; r++) sacc = fma(lv[r], xk[r0 + r], sacc);
            }
            ywork[c] -= sacc;
        }
        if (kb > 0) {                       // rows of step kb - 1 (a full block: only the last one can be partial)
            const int k1 = k0 - NB;
#pragma unroll
            for (int r = 0; r < NB; r++) l[r] = (tid < k1) ? A[(size_t) (k1 + r) * ld + tid] : 0.0;
        }
        // no barrier here: xk is rewritten only behind the next step's first barrier, ys / Li were last read before this step's
        // second one, and ywork[c] is only ever touched by thread c mod 512
    }
}

// symmetric S (both triangles filled by the Schur kernel) + E in row n.  x receives the solution.  band: see chol_solve_large.
// Lmat: (n+1) x n factor matrix (out of place: A's panel columns stay readable during a step).
// linv_ws: ceil(n/32) * 1024 doubles (+ n doubles of back-substitution workspace behind it).
int chol_solve(cudaStream_t st, double *A, double *Lmat, int n, double *linv_ws, double *x, Scalars *sc, const CholBand *band)
{
    const int nbk = (n + NB - 1) / NB;
    if (n > CHOL_LARGE_MIN) return chol_solve_large(st, A, Lmat, n, linv_ws, linv_ws + (size_t) nbk * NB * NB, x, sc, band);
    if (n > LNB) {      // small systems: one co-resident dataflow launch per factorisation (ba_chol_dataflow.cu)
        bool used = false;
        int rc = chol_solve_dataflow(st, A, Lmat, n, linv_ws, x, sc, &used);
        if (rc != BSFM_OK || used) return rc;
    }
    const int ld = n;
    double *ywork = linv_ws + (size_t) nbk * NB * NB;
    // one fused chol_step launch per 32 columns over the whole trailing matrix
    for (int k = 0; k < nbk; k++) {
        int tiles = 0;
        for (int c = k + 1; c < nbk; c++) tiles += nbk - c + 1;
        if (tiles > 800) {
            // many more tiles than resident CTAs: factor the diagonal block once, then the GEMM-style tile kernel
            chol_step_kernel<<<1, CST, 0, st>>>(A, Lmat, ld, n, k, k + 1, linv_ws, sc);
            BSFM_KERNEL_CHECK();
            chol_tile_kernel<<<tiles, 256, 0, st>>>(A, Lmat, ld, n, k, nbk, linv_ws);
            BSFM_KERNEL_CHECK();
        } else {
            BSFM_CUDA_TRY(launch_pdl(chol_step_kernel, dim3(1 + tiles), dim3(CST), st, A, Lmat, ld, n, k, nbk, linv_ws, sc));
            count_launch();
        }
    }
    BSFM_CUDA_TRY(launch_pdl(chol_backsolve_blocked_kernel, dim3(1), dim3(512), st, (const double *) Lmat, ld, n, (const double *) linv_ws, x, ywork));
    count_launch();
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm
