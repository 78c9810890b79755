// match_kernels.cu -- sm_90a kernels of the MATCH hot path.  See match_kernels.cuh for layout.
#include "match_kernels.cuh"
#include "tc_ptx.cuh"
#include <climits>

namespace bsfm {
namespace match {

// ---------------------------------------------------------------------------------------------
// prep: raw host-order descriptors (n_i x 128 per image, concatenated) -> squared norms (for the per-image
// sort), then the padded, norm-sorted, swizzled layout.  One warp per row; lane l handles bytes [4l, 4l+4).
// ---------------------------------------------------------------------------------------------
__global__ void raw_norm_kernel(const uint8_t *__restrict__ raw, int64_t total_keys, int32_t *__restrict__ norms_raw, int32_t *__restrict__ iota)
{
    const int64_t row = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= total_keys) return;
    const uint8_t *src = raw + row * DESC_BYTES + lane * 4;
    const uint32_t w = (uint32_t) src[0] | ((uint32_t) src[1] << 8) | ((uint32_t) src[2] << 16) | ((uint32_t) src[3] << 24);
    uint32_t s = __dp4a(w, w, 0u);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) { norms_raw[row] = (int32_t) s; iota[row] = (int32_t) row; }
}

// sorted_src[key_off[img] + pos] = raw row (global) that is the pos-th smallest-norm key of image img
__global__ void prep_kernel(const uint8_t *__restrict__ raw, const int64_t *__restrict__ key_off,
                            const int32_t *__restrict__ img_doff, const int32_t *__restrict__ tile_img,
                            const int32_t *__restrict__ sorted_src, const int32_t *__restrict__ sorted_norms,
                            uint8_t *__restrict__ keys_sw, int32_t *__restrict__ norms, int32_t *__restrict__ perm,
                            int64_t row_begin, int64_t row_end, int64_t key_base)
{
    // rows [row_begin, row_end) of the device layout; `raw`, `sorted_src`, `sorted_norms` hold the keys [key_base, ...) only
    // (a rank of a sharded build prepares its own images; key_base = 0 and the whole row range otherwise)
    int64_t row = row_begin + (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= row_end) return;
    int img = tile_img[row >> 7];
    uint32_t w = 0;
    int32_t nrm = NORM_PAD, orig = -1;
    if (img >= 0) {
        int64_t k = row - img_doff[img];
        int64_t n = key_off[img + 1] - key_off[img];
        if (k < n) {
            const int64_t srow = sorted_src[key_off[img] - key_base + k];      // row inside `raw`
            const uint8_t *src = raw + srow * DESC_BYTES + lane * 4;
            w = (uint32_t) src[0] | ((uint32_t) src[1] << 8) | ((uint32_t) src[2] << 16) | ((uint32_t) src[3] << 24);
            nrm = sorted_norms[key_off[img] - key_base + k];
            orig = (int32_t) (srow + key_base - key_off[img]);
        }
    }
    int c = lane >> 2;  // 16-byte chunk
    uint32_t *dst = reinterpret_cast<uint32_t *>(keys_sw + sw_chunk_offset(row, c)) + (lane & 3);
    *dst = w;
    if (lane == 0) { norms[row] = nrm; perm[row] = orig; }
}

// ---------------------------------------------------------------------------------------------
// DP4A kernel: one CTA per work unit (128 query rows x whole database image).  CUDA-core second
// implementation used to cross-check the tensor-core kernel at full size and as the selectable
// BSFM_MATCH_KERNEL_DP4A path.  Exact top-2 with index per row; emits final matches directly.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void top2_insert(int &m1, int &m2, int &mi, int t, int idx, bool ties, const int32_t *perm_img)
{
    // keeps (m1 <= m2); a thread sees its columns in ascending norm-sorted position, so without `ties` the first seen wins a
    // tie.  With `ties` (a tie can pass the ratio test) a tied column replaces the best when its caller index is smaller.
    if (t < m1) { m2 = m1; m1 = t; mi = idx; }
    else {
        if (t < m2) m2 = t;
        if (ties && t == m1 && perm_img[idx] < perm_img[mi]) mi = idx;
    }
}

__global__ void __launch_bounds__(256) match_dp4a_kernel(MatchParams P)
{
    __shared__ uint32_t sQ[32][TILE_Q];
    __shared__ uint32_t sD[32][128];
    __shared__ int32_t sN[128];

    const int u = P.unit_begin + blockIdx.x;
    if (u >= P.unit_end) return;
    const int k = find_run_image(P.run_imgs, P.num_run_imgs, u);
    const RunImage R = P.run_imgs[k];
    const int64_t a_row0 = (int64_t) (R.atile0 + (u - R.unit0)) * TILE_Q;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const bool ties = P.ties_pass != 0;
    const int32_t *perm_img = P.perm + R.db_row0;   // norm-sorted position of image R -> caller index

    // query tile -> sQ[k4][row]
    for (int idx = tid; idx < TILE_Q * 8; idx += 256) {
        int c = idx >> 7, row = idx & 127;
        uint4 v = *reinterpret_cast<const uint4 *>(P.keys_sw + sw_chunk_offset(a_row0 + row, c));
        sQ[c * 4 + 0][row] = v.x; sQ[c * 4 + 1][row] = v.y; sQ[c * 4 + 2][row] = v.z; sQ[c * 4 + 3][row] = v.w;
    }

    int m1[8], m2[8], mi[8];
#pragma unroll
    for (int a = 0; a < 8; a++) { m1[a] = INT_MAX; m2[a] = INT_MAX; mi[a] = -1; }

    const int ntiles = R.ntiles_db * 2;  // 128-row database tiles
    for (int tile = 0; tile < ntiles; tile++) {
        const int64_t d_row0 = (int64_t) R.db_row0 + (int64_t) tile * 128;
        __syncthreads();
        for (int idx = tid; idx < 128 * 8; idx += 256) {
            int c = idx >> 7, row = idx & 127;
            uint4 v = *reinterpret_cast<const uint4 *>(P.keys_sw + sw_chunk_offset(d_row0 + row, c));
            sD[c * 4 + 0][row] = v.x; sD[c * 4 + 1][row] = v.y; sD[c * 4 + 2][row] = v.z; sD[c * 4 + 3][row] = v.w;
        }
        if (tid < 128) sN[tid] = P.norms[d_row0 + tid];
        __syncthreads();

        uint32_t acc[8][8];
#pragma unroll
        for (int a = 0; a < 8; a++)
#pragma unroll
            for (int b = 0; b < 8; b++) acc[a][b] = 0;
#pragma unroll 4
        for (int k4 = 0; k4 < 32; k4++) {
            uint32_t q[8], d[8];
#pragma unroll
            for (int a = 0; a < 8; a++) q[a] = sQ[k4][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 8; b++) d[b] = sD[k4][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 8; a++)
#pragma unroll
                for (int b = 0; b < 8; b++) acc[a][b] = __dp4a(q[a], d[b], acc[a][b]);
        }
#pragma unroll
        for (int b = 0; b < 8; b++) {
            const int col = tile * 128 + tx + 16 * b;
            const int nb = sN[tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 8; a++) {
                int t = nb - 2 * (int) acc[a][b];
                top2_insert(m1[a], m2[a], mi[a], t, col, ties, perm_img);
            }
        }
    }

    // merge the 16 column-threads of every row (lanes differing in the low 4 bits); of two tied bests the smaller caller
    // index wins, so the result does not depend on the shuffle tree
#pragma unroll
    for (int a = 0; a < 8; a++) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            int o1 = __shfl_xor_sync(0xffffffffu, m1[a], o);
            int o2 = __shfl_xor_sync(0xffffffffu, m2[a], o);
            int oi = __shfl_xor_sync(0xffffffffu, mi[a], o);
            int hi = max(m1[a], o1);
            int lo2 = min(m2[a], o2);
            if (o1 < m1[a] || (o1 == m1[a] && perm_img[oi] < perm_img[mi[a]])) mi[a] = oi;
            m1[a] = min(m1[a], o1);
            m2[a] = min(hi, lo2);
        }
    }
    if (tx == 0) {
#pragma unroll
        for (int a = 0; a < 8; a++) {
            const int r = ty + 16 * a;
            const int na = P.norms[a_row0 + r];
            if (na >= NORM_PAD_HALF) continue;  // padding query row
            const int d0 = na + m1[a];
            const int d1 = (m2[a] >= NORM_PAD_HALF) ? INT_MAX : na + m2[a];
            if (ratio_pass(P, d0, d1)) {
                int pos = atomicAdd(&P.counters[1], 1);
                if (pos < P.match_cap) {
                    P.match_slot[pos] = match_sort_key(P, R, a_row0 + r);
                    P.match_idx2[pos] = mi[a];
                } else {
                    P.counters[2] = 1;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// wgmma kernel: persistent, warp-specialised (variants: match_tc_body below).
//   warps 0..7 : two consumer warpgroups; warpgroup g owns query rows [64 g, 64 g + 64) of every unit, issues its own
//                wgmma.mma_async (u8 x u8 -> s32, M64 N128 K32 x4 per half tile) and reduces the accumulators in registers
//   warp 8     : TMA producer (cp.async.bulk, one 16 KB query tile per unit, 32 KB database tiles)
// Every 256-row database tile is computed as two N = 128 halves into two register accumulators: the MMAs of the second
// half run while the first half is reduced.  Shared-memory database ring of 4 stages, query tile double-buffered.
// A thread holds rows r0 = 16 w + g and r0 + 8 of its warpgroup (lane = 4 g + q) and two of every 8 columns; the four
// lanes of a quad together hold a whole row, so a chunk reduction is a thread-local tree plus two shuffles.
// Epilogue per element: t = |p|^2 - 2*dot, chunk minimum (exact mode) or chunk maximum of the dot products (bound mode).
// Per chunk the row keeps (m1 = smallest chunk-min, s2 = second smallest chunk-min, bchunk).  d0 is exact; d1 is bounded
// above by s2, so only rows passing the ratio test with that bound can match: they are pushed as candidates and resolved
// exactly by match_verify_kernel.
// ---------------------------------------------------------------------------------------------

using namespace bsfm::ptx;   // tc_ptx.cuh

struct UnitInfo {
    int64_t a_row0;
    int32_t db_row0, n, ntiles_db;
};
// Work units of a CTA ascend, and most consecutive units stay inside the same run image: every role keeps a cursor
// (the image's unit range and fields in registers) and only touches global memory when a unit leaves the image --
// a binary search per unit would put a chain of dependent global loads on the producer's critical path.
struct UnitCursor {
    int32_t k = -1, unit0 = 0, unit_end = 0;      // current run image and its unit range [unit0, unit_end)
    int32_t atile0 = 0, db_row0 = 0, n = 0, ntiles_db = 0;
};
__device__ __forceinline__ void cursor_load(const MatchParams &P, UnitCursor &c)
{
    const RunImage *R = P.run_imgs + c.k;
    c.unit0 = R->unit0; c.unit_end = R->unit0 + R->nunits;
    c.atile0 = R->atile0; c.db_row0 = R->db_row0; c.n = R->n; c.ntiles_db = R->ntiles_db;
}
__device__ __forceinline__ UnitInfo decode_unit(const MatchParams &P, UnitCursor &c, int u)
{
    if (c.k < 0 || u >= c.unit_end) {
        if (c.k >= 0 && c.k + 1 < P.num_run_imgs) { c.k++; cursor_load(P, c); }       // usually the next image
        if (c.k < 0 || u < c.unit0 || u >= c.unit_end) { c.k = find_run_image(P.run_imgs, P.num_run_imgs, u); cursor_load(P, c); }
    }
    UnitInfo U;
    U.a_row0 = (int64_t) (c.atile0 + (u - c.unit0)) * TILE_Q;
    U.db_row0 = c.db_row0;
    U.n = c.n;
    U.ntiles_db = c.ntiles_db;
    return U;
}

// state of one query row across the database image
struct RowState {
    // exact mode : m1 = smallest chunk-min of t, s2 = second smallest chunk-min, bchunk.
    // bound mode : m1 = smallest chunk LOWER bound, s2 = second smallest lower bound,
    //              ubb = UPPER bound of the best chunk, uo = smallest upper bound of the others.
    int m1 = INT_MAX, s2 = INT_MAX, bchunk = 0, ubb = INT_MAX, uo = INT_MAX;
};
__device__ __forceinline__ int quad_max(int v)
{
    v = max(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return max(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ int quad_min(int v)
{
    v = min(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return min(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// reduces the 64 x W accumulator of the columns [col0, col0 + W) of the database image into the two rows' states
template <bool BOUND, int W>
__device__ __forceinline__ void reduce_part(const MatchParams &P, const uint32_t (&d)[W / 2], int col0, int q, int db_row0,
                                            const int *sNall, RowState &s0, RowState &s1)
{
    const int neg2 = P.neg2;     // runtime -2: keeps the multiply-add on the FMA pipe (IMAD)
    if constexpr (BOUND) {
        // keys are norm-sorted inside an image, so a chunk's norms span [norm(first), norm(last)] and  min_c t  lies in
        // [nbmin - 2 vmax, nbmax - 2 vmax]  with vmax the chunk's largest dot product: the hot loop is a bare MAX tree
#pragma unroll
        for (int c = 0; c < W / BCHUNK; c++) {
            int v0 = 0, v1 = 0;
#pragma unroll
            for (int j = c * (BCHUNK / 8); j < (c + 1) * (BCHUNK / 8); j++) {
                v0 = max(max((int) d[4 * j + 0], (int) d[4 * j + 1]), v0);
                v1 = max(max((int) d[4 * j + 2], (int) d[4 * j + 3]), v1);
            }
            v0 = quad_max(v0); v1 = quad_max(v1);
            const int c0 = col0 + c * BCHUNK;
            const int chunk_id = c0 / BCHUNK;
            const int nlo = sNall[c0], nhi = sNall[c0 + BCHUNK - 1];
            auto bookkeep = [&](RowState &s, int vmax) {
                const int lb = vmax * neg2 + nlo;
                const int ub = vmax * neg2 + nhi;
                const bool nb_best = lb < s.m1;
                s.s2 = nb_best ? s.m1 : min(s.s2, lb);
                s.uo = min(s.uo, nb_best ? s.ubb : ub);
                s.ubb = nb_best ? ub : s.ubb;
                s.bchunk = nb_best ? chunk_id : s.bchunk;
                s.m1 = min(s.m1, lb);
            };
            bookkeep(s0, v0);
            bookkeep(s1, v1);
        }
    } else {
        const int *nb = P.norms + (size_t) db_row0 + col0 + 2 * q;
#pragma unroll
        for (int c = 0; c < W / CHUNK; c++) {
            int c0 = INT_MAX, c1 = INT_MAX;
#pragma unroll
            for (int j = c * (CHUNK / 8); j < (c + 1) * (CHUNK / 8); j++) {
                const int2 n2 = __ldg(reinterpret_cast<const int2 *>(nb + 8 * j));
                c0 = min(min((int) d[4 * j + 0] * neg2 + n2.x, (int) d[4 * j + 1] * neg2 + n2.y), c0);
                c1 = min(min((int) d[4 * j + 2] * neg2 + n2.x, (int) d[4 * j + 3] * neg2 + n2.y), c1);
            }
            c0 = quad_min(c0); c1 = quad_min(c1);
            const int chunk_id = col0 / CHUNK + c;
            auto update = [&](RowState &s, int cm) {
                // (m1, s2) <- two smallest of {m1, s2, cm}
                const int hi = max(s.m1, cm);
                if (cm < s.m1) s.bchunk = chunk_id;
                s.m1 = min(s.m1, cm);
                s.s2 = min(s.s2, hi);
            };
            update(s0, c0);
            update(s1, c1);
        }
    }
}

// waits until at most n of this warpgroup's committed MMA groups are still in flight (n is a constant after unrolling)
__device__ __forceinline__ void wgmma_wait_upto(int n)
{
    if (n >= 3) wgmma_wait<3>();
    else if (n == 2) wgmma_wait<2>();
    else if (n == 1) wgmma_wait<1>();
    else wgmma_wait<0>();
}

// BOUND = true : bound epilogue (every database image of the launch fits the norm staging buffer)
// BOUND = false: exact chunk-minimum epilogue (any image size)
// QUAD = true  : (bound epilogue) every 256-row database tile is computed as FOUR N = 64 parts into four register accumulators
//                instead of two N = 128 halves: the MMAs of parts p+1.. run while part p is reduced, so more of the epilogue
//                overlaps the tensor core
// PAIR = true  : (bound epilogue) two CTAs of a cluster take two query units of the same database image and share every database
//                tile: each CTA loads HALF of it and multicasts it into both CTAs' shared memory (TMA multicast), which halves the
//                L2 -> SM traffic per MAC.  A stage is refilled only when the consumers of BOTH CTAs have released it.
template <bool BOUND, bool QUAD, bool PAIR>
__device__ __forceinline__ void match_tc_body(const MatchParams &P)
{
    static_assert(!(QUAD || PAIR) || BOUND, "the four-part and CTA-pair variants exist for the bound epilogue");
    constexpr int NPARTS = QUAD ? 4 : 2;            // accumulator parts per database tile
    constexpr int W = TILE_DB / NPARTS;              // columns per part
    extern __shared__ uint8_t smem_raw[];
    // manual 1024-byte alignment (SWIZZLE_128B atoms); the same offsets in both CTAs of a pair
    const uint32_t raw_addr = smem_u32(smem_raw);
    const uint32_t base = (raw_addr + 1023u) & ~1023u;
    uint8_t *smem = smem_raw + (base - raw_addr);

    const uint32_t sA = base + TC_SMEM_A;
    const uint32_t sB = base + TC_SMEM_B;
    const uint32_t bar0 = base + TC_SMEM_BAR;
    constexpr int MATH_WARPS = TC_MATH_THREADS / 32;
    const uint32_t bar_b_full = bar0;                            // [TC_B_STAGES]
    const uint32_t bar_b_empty = bar0 + 8 * TC_B_STAGES;         // [TC_B_STAGES]
    const uint32_t bar_a_full = bar0 + 16 * TC_B_STAGES;         // [2]
    const uint32_t bar_a_empty = bar_a_full + 16;                // [2]
    static_assert(8 * (2 * TC_B_STAGES + 4) <= 256, "barrier region");
    const uint32_t crank = PAIR ? cluster_ctarank() : 0u;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_B_STAGES; s++) { mbar_init(bar_b_full + 8 * s, 1); mbar_init(bar_b_empty + 8 * s, (PAIR ? 2 : 1) * MATH_WARPS); }
        for (int s = 0; s < 2; s++) { mbar_init(bar_a_full + 8 * s, 1); mbar_init(bar_a_empty + 8 * s, MATH_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();      // the peer's barriers must be initialised before any multicast or remote arrive

    // pair mode: cluster c takes the unit pairs (2c, 2c+1), (2c + G, 2c + 1 + G), ...: both units of a pair share the database
    // image (images are padded to 256 rows, so every image contributes an even number of 128-row query units)
    const int u_first = PAIR ? P.unit_begin + 2 * (int) (blockIdx.x >> 1) + (int) crank : P.unit_begin + (int) blockIdx.x;
    const int u_step = PAIR ? (int) (gridDim.x & ~1u) : (int) gridDim.x;

    if (warp == MATH_WARPS) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            uint32_t bs = 0, bph = 0, as = 0, aph = 0;
            UnitCursor cur;
            for (int u = u_first; u < P.unit_end; u += u_step) {
                const UnitInfo U = decode_unit(P, cur, u);
                mbar_wait_backoff(bar_a_empty + 8 * as, aph ^ 1);
                mbar_expect_tx(bar_a_full + 8 * as, TC_A_BYTES);
                tma_bulk_g2s(sA + as * TC_A_BYTES, P.keys_sw + (size_t) U.a_row0 * DESC_BYTES, TC_A_BYTES, bar_a_full + 8 * as);
                as ^= 1; if (as == 0) aph ^= 1;
                const uint8_t *src = P.keys_sw + (size_t) U.db_row0 * DESC_BYTES;
                for (int t = 0; t < U.ntiles_db; t++) {
                    mbar_wait_backoff(bar_b_empty + 8 * bs, bph ^ 1);
                    mbar_expect_tx(bar_b_full + 8 * bs, TC_B_BYTES);      // pair: both halves land here, one from each CTA
                    if (PAIR) {
                        constexpr uint32_t HALF = TC_B_BYTES / 2;
                        tma_bulk_g2s_multicast(sB + bs * TC_B_BYTES + crank * HALF, src + (size_t) t * TC_B_BYTES + crank * HALF, HALF,
                                               bar_b_full + 8 * bs, (uint16_t) 3);
                    } else {
                        tma_bulk_g2s(sB + bs * TC_B_BYTES, src + (size_t) t * TC_B_BYTES, TC_B_BYTES, bar_b_full + 8 * bs);
                    }
                    if (++bs == TC_B_STAGES) { bs = 0; bph ^= 1; }
                }
            }
        }
    } else {
    // ===================== consumer warpgroups =====================
    const int wg = warp >> 2;                       // query rows [64 wg, 64 wg + 64) of the unit
    const int g = lane >> 2, q = lane & 3;
    const int row0 = 64 * wg + 16 * (warp & 3) + g;  // and row0 + 8
    int *sNall = reinterpret_cast<int *>(smem + TC_SMEM_NALL);
    int staged_row0 = -1;
    uint32_t bs = 0, bph = 0, as = 0, aph = 0;
    UnitCursor cur;
    for (int u = u_first; u < P.unit_end; u += u_step) {
        const UnitInfo U = decode_unit(P, cur, u);
        // Database norms (bound mode): the host guarantees that every image fits (<= TC_NORM_CAP rows); they are staged
        // ONCE per (CTA, database image) -- consecutive units of a CTA share the image -- so the tile loop has no barrier
        if (BOUND && staged_row0 != U.db_row0) {
            asm volatile("bar.sync 1, %0;" ::"n"(TC_MATH_THREADS) : "memory");   // everyone done with the old image
            for (int i = threadIdx.x; i < U.ntiles_db * TILE_DB; i += TC_MATH_THREADS) sNall[i] = P.norms[(size_t) U.db_row0 + i];
            asm volatile("bar.sync 1, %0;" ::"n"(TC_MATH_THREADS) : "memory");
            staged_row0 = U.db_row0;
        }
        RowState s0, s1;
        mbar_wait(bar_a_full + 8 * as, aph);
        const uint64_t adesc = make_sw128_desc(sA + as * TC_A_BYTES + wg * (64 * DESC_BYTES));
        for (int t = 0; t < U.ntiles_db; t++) {
            mbar_wait(bar_b_full + 8 * bs, bph);
            const uint64_t bdesc = make_sw128_desc(sB + bs * TC_B_BYTES);
            uint32_t d[NPARTS][W / 2];
            wgmma_fence();
#pragma unroll
            for (int p = 0; p < NPARTS; p++) {
                // K = 4 x 32 bytes: +32 B = +2 in the descriptor start field; part p starts W rows x 128 B = 8 W further
#pragma unroll
                for (int kk = 0; kk < 4; kk++) {
                    const uint64_t bd = bdesc + (uint64_t) (p * W * 8 + kk * 2);
                    if constexpr (W == 128) wgmma_u8_n128(d[p], adesc + (uint64_t) (kk * 2), bd, kk > 0);
                    else wgmma_u8_n64(d[p], adesc + (uint64_t) (kk * 2), bd, kk > 0);
                }
                wgmma_commit();
            }
#pragma unroll
            for (int p = 0; p < NPARTS; p++) {
                wgmma_wait_upto(NPARTS - 1 - p);
                wgmma_fence_regs(d[p]);
                if (p == NPARTS - 1) {
                    // the shared-memory operands are consumed: hand the stage (and after the last tile the query tile) back;
                    // pair mode: the stage is refilled in both CTAs, so the release goes to both
                    __syncwarp();
                    if (lane == 0) {
                        if (PAIR) { mbar_arrive_cluster(bar_b_empty + 8 * bs, 0); mbar_arrive_cluster(bar_b_empty + 8 * bs, 1); }
                        else mbar_arrive(bar_b_empty + 8 * bs);
                        if (t + 1 == U.ntiles_db) mbar_arrive(bar_a_empty + 8 * as);
                    }
                    if (++bs == TC_B_STAGES) { bs = 0; bph ^= 1; }
                }
                reduce_part<BOUND, W>(P, d[p], t * TILE_DB + p * W, q, U.db_row0, sNall, s0, s1);
            }
        }
        as ^= 1; if (as == 0) aph ^= 1;

        // candidate decision of both rows; the four lanes of a quad hold identical states, lane q = 0 reports
        bool cand[2] = {false, false};
        int f5[2] = {INT_MAX, INT_MAX}, f6[2] = {INT_MAX, INT_MAX};
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const RowState &s = r ? s1 : s0;
            const int na = P.norms[U.a_row0 + row0 + 8 * r];
            if (q != 0 || na >= NORM_PAD_HALF) continue;
            if (BOUND) {
                // two distinct keys with t <= max(ubb, uo) exist, so d1 <= na + max(ubb, uo); d0 >= na + m1
                const int ubs = max(s.ubb, s.uo);
                const int d1u = (ubs >= NORM_PAD_HALF) ? INT_MAX : na + ubs;
                cand[r] = (double) (na + s.m1) < P.ratio_sq * (double) d1u;
                f5[r] = s.s2; f6[r] = s.uo;
            } else {
                // exact d0, upper bound on d1
                const int d0 = na + s.m1;
                const int d1u = (s.s2 >= NORM_PAD_HALF) ? INT_MAX : na + s.s2;
                cand[r] = (double) d0 < P.ratio_sq * (double) d1u;
                f5[r] = d1u;
            }
        }
        const unsigned b0 = __ballot_sync(0xffffffffu, cand[0]), b1 = __ballot_sync(0xffffffffu, cand[1]);
        if (b0 | b1) {
            int basepos = 0;
            if (lane == 0) basepos = atomicAdd(&P.counters[0], __popc(b0) + __popc(b1));
            basepos = __shfl_sync(0xffffffffu, basepos, 0);
#pragma unroll
            for (int r = 0; r < 2; r++) {
                if (!cand[r]) continue;
                const RowState &s = r ? s1 : s0;
                const int pos = basepos + (r ? __popc(b0) : 0) + __popc((r ? b1 : b0) & ((1u << lane) - 1u));
                if (pos < P.cand_cap) {
                    constexpr int CW = BOUND ? BCHUNK : CHUNK;   // width of the chunk the verify kernel recomputes
                    const int row = row0 + 8 * r;
                    const int col0 = s.bchunk * CW;
                    const size_t cap = (size_t) P.cand_cap;
                    P.cand[0 * cap + pos] = (u - P.unit_begin) * TILE_Q + row;
                    P.cand[1 * cap + pos] = (int32_t) (U.a_row0 + row);
                    P.cand[2 * cap + pos] = U.db_row0 + col0;
                    P.cand[3 * cap + pos] = col0;
                    P.cand[4 * cap + pos] = min(CW, U.n - col0);
                    P.cand[5 * cap + pos] = f5[r];
                    P.cand[6 * cap + pos] = BOUND ? f6[r] : INT_MIN;   // INT_MIN marks an exact-mode candidate
                } else {
                    P.counters[2] = 1;
                }
            }
        }
    }
    }
    // pair mode: neither CTA may leave while the peer's multicast copies into its shared memory or its remote arrives are in flight
    if (PAIR) cluster_sync_all();
}

__global__ void __launch_bounds__(TC_THREADS, 1) match_tc_kernel(MatchParams P) { match_tc_body<false, false, false>(P); }
__global__ void __launch_bounds__(TC_THREADS, 1) match_tc_bound_kernel(MatchParams P) { match_tc_body<true, false, false>(P); }
__global__ void __launch_bounds__(TC_THREADS, 1) match_tc_quad_kernel(MatchParams P) { match_tc_body<true, true, false>(P); }
// launched with cluster dimension (2, 1, 1)
__global__ void __launch_bounds__(TC_THREADS, 1) match_tc_pair_kernel(MatchParams P) { match_tc_body<true, false, true>(P); }

// ---------------------------------------------------------------------------------------------
// verify: one warp per candidate.  Recomputes the 32 distances of the winning chunk with the
// DEFINITION (sum of squared differences, kd_pr_search.cpp:200-209), finds the exact nearest
// column and the chunk's own second minimum, applies the final ratio test.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int sqdist_rows(const uint8_t *keys_sw, int64_t ra, int64_t rb)
{
    uint32_t acc = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) {
        const uint4 a = *reinterpret_cast<const uint4 *>(keys_sw + sw_chunk_offset(ra, c));
        const uint4 b = *reinterpret_cast<const uint4 *>(keys_sw + sw_chunk_offset(rb, c));
        uint32_t dx = __vabsdiffu4(a.x, b.x), dy = __vabsdiffu4(a.y, b.y), dz = __vabsdiffu4(a.z, b.z), dw = __vabsdiffu4(a.w, b.w);
        acc = __dp4a(dx, dx, acc); acc = __dp4a(dy, dy, acc); acc = __dp4a(dz, dz, acc); acc = __dp4a(dw, dw, acc);
    }
    return (int) acc;
}

__global__ void __launch_bounds__(256) match_verify_kernel(MatchParams P, int ncand)
{
    const int w = (int) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= ncand) return;
    const size_t cap = (size_t) P.cand_cap;
    const int slot = P.cand[0 * cap + w];
    const int qrow = P.cand[1 * cap + w];
    const int db0 = P.cand[2 * cap + w];
    const int col0 = P.cand[3 * cap + w];
    const int nvalid = P.cand[4 * cap + w];
    const int f5 = P.cand[5 * cap + w];
    const int f6 = P.cand[6 * cap + w];

    // up to 64 rows per candidate (bound chunks may be 64 wide): two distances per lane, lane-local top-2 first.
    // (m1, mk) orders by distance, then by caller index: of keys tied for the nearest distance the smallest caller index wins
    int m1 = INT_MAX, m2 = INT_MAX, mi = lane, mk = INT_MAX;
    if (lane < nvalid) { m1 = sqdist_rows(P.keys_sw, qrow, (int64_t) db0 + lane); mk = P.perm[db0 + lane]; }
    if (lane + 32 < nvalid) {
        const int d = sqdist_rows(P.keys_sw, qrow, (int64_t) db0 + lane + 32);
        const int k = P.perm[db0 + lane + 32];
        if (d < m1 || (d == m1 && k < mk)) { m2 = m1; m1 = d; mi = lane + 32; mk = k; } else m2 = d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        int o1 = __shfl_xor_sync(0xffffffffu, m1, o);
        int o2 = __shfl_xor_sync(0xffffffffu, m2, o);
        int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        int ok = __shfl_xor_sync(0xffffffffu, mk, o);
        int hi = max(m1, o1);
        int lo2 = min(m2, o2);
        if (o1 < m1 || (o1 == m1 && ok < mk)) { mi = oi; mk = ok; }
        m1 = min(m1, o1);
        m2 = min(hi, lo2);
    }
    if (lane == 0) {
        bool match = false, hard = false;
        if (f6 == INT_MIN) {
            // exact mode: d0 = m1 is the global minimum, f5 bounds d1 from above through the other chunks.  f5 == m1 means
            // another chunk holds a key at distance d0: when such a tie can pass, the full scan picks among all tied keys
            const int d1 = min(f5, m2);
            if (P.ties_pass && f5 == m1) hard = true;
            else match = ratio_pass(P, m1, d1);
        } else {
            // bound mode: the chunk with the smallest lower bound was recomputed exactly (m1, m2).  It holds the
            // global minimum iff m1 <= every other chunk's lower bound; d1 lies in [min(m2, L2), min(m2, Uo)].
            // m1 == L2 leaves open a key of another chunk at distance d0: undecided when such a tie can pass
            const int na = P.norms[qrow];
            const int l2d = (f5 >= NORM_PAD_HALF) ? INT_MAX : na + f5;
            const int uod = (f6 >= NORM_PAD_HALF) ? INT_MAX : na + f6;
            if (m1 > l2d || (P.ties_pass && m1 == l2d)) hard = true;
            else {
                const int d1_low = min(m2, l2d), d1_up = min(m2, uod);
                if (ratio_pass(P, m1, d1_low)) match = true;
                else if (ratio_pass(P, m1, d1_up)) hard = true;   // undecided inside the bound slack
            }
        }
        if (hard) {
            int pos = atomicAdd(&P.counters[3], 1);
            if (pos < P.cand_cap) { P.hard[pos] = slot; P.hard[(size_t) P.cand_cap + pos] = qrow; }
            else P.counters[2] = 1;
        }
        if (match) {
            int pos = atomicAdd(&P.counters[1], 1);
            if (pos < P.match_cap) {
                const int u = P.unit_begin + (slot >> 7);
                const RunImage R = P.run_imgs[find_run_image(P.run_imgs, P.num_run_imgs, u)];
                P.match_slot[pos] = match_sort_key(P, R, qrow);
                P.match_idx2[pos] = col0 + mi;
            } else {
                P.counters[2] = 1;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// full scan: one block per "hard" row (bounds undecided): exact two nearest keys over the whole database
// image with the definition, final ratio test.  Rare by construction.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) match_fullscan_kernel(MatchParams P, int nhard)
{
    // one 256-thread block per hard row: every warp scans a strided eighth of the image, then the warps' top-2 merge
    __shared__ int s_m1[8], s_m2[8], s_mi[8], s_mk[8];
    const int w = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (w >= nhard) return;
    const int slot = P.hard[w];
    const int qrow = P.hard[(size_t) P.cand_cap + w];
    const int u = P.unit_begin + (slot >> 7);
    const RunImage R = P.run_imgs[find_run_image(P.run_imgs, P.num_run_imgs, u)];
    // (m1, mk) orders by distance, then by caller index: of keys tied for the nearest distance the smallest caller index wins
    int m1 = INT_MAX, m2 = INT_MAX, mi = INT_MAX, mk = INT_MAX;
    for (int c = threadIdx.x; c < R.n; c += 256) {
        const int d = sqdist_rows(P.keys_sw, qrow, (int64_t) R.db_row0 + c);
        const int k = P.perm[(int64_t) R.db_row0 + c];
        if (d < m1 || (d == m1 && k < mk)) { m2 = m1; m1 = d; mi = c; mk = k; } else if (d < m2) m2 = d;
    }
    auto merge = [&](int o1, int o2, int oi, int ok) {
        const int hi = max(m1, o1);
        const int lo2 = min(m2, o2);
        if (o1 < m1 || (o1 == m1 && ok < mk)) { mi = oi; mk = ok; }
        m1 = min(m1, o1);
        m2 = min(hi, lo2);
    };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int o1 = __shfl_xor_sync(0xffffffffu, m1, o);
        const int o2 = __shfl_xor_sync(0xffffffffu, m2, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        const int ok = __shfl_xor_sync(0xffffffffu, mk, o);
        merge(o1, o2, oi, ok);
    }
    if (lane == 0) { s_m1[warp] = m1; s_m2[warp] = m2; s_mi[warp] = mi; s_mk[warp] = mk; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int q = 1; q < 8; q++) merge(s_m1[q], s_m2[q], s_mi[q], s_mk[q]);
        if (ratio_pass(P, m1, m2)) {
            int pos = atomicAdd(&P.counters[1], 1);
            if (pos < P.match_cap) { P.match_slot[pos] = match_sort_key(P, R, qrow); P.match_idx2[pos] = mi; }
            else P.counters[2] = 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// finalize: sorted (slot, idx2) -> (idx1, idx2) records + per-pair counts.
// ---------------------------------------------------------------------------------------------
__global__ void match_finalize_kernel(const uint32_t *__restrict__ slots, const int32_t *__restrict__ idx2,
                                      int nmatch, const RunImage *__restrict__ run_imgs, int K, int unit_begin,
                                      const int32_t *__restrict__ tile_img, const int32_t *__restrict__ img_doff,
                                      const int32_t *__restrict__ perm,
                                      int32_t *__restrict__ out_pairs /* [nmatch][2] */,
                                      int32_t *__restrict__ pair_counts)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nmatch) return;
    const uint32_t slot = slots[e];
    const int u = unit_begin + (int) (slot >> 7);
    const int r = (int) (slot & 127u);
    const int k = find_run_image(run_imgs, K, u);
    const RunImage R = run_imgs[k];
    const int atile = R.atile0 + (u - R.unit0);
    const int j = tile_img[atile];
    const int idx1 = atile * TILE_Q + r - img_doff[j];
    out_pairs[2 * (size_t) e + 0] = idx1;
    out_pairs[2 * (size_t) e + 1] = perm[(size_t) R.db_row0 + idx2[e]];   // norm-sorted position -> caller's key index
    atomicAdd(&pair_counts[R.pair0 + (j - R.start_img)], 1);
}

}  // namespace match
}  // namespace bsfm
