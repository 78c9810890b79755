// ba_order.cu -- camera order of large reduced camera systems (host only, once per solve).
//
// The large Cholesky (ba_chol_large.cu) skips the 128 x 128 tiles of the trailing update whose panel blocks are exactly zero,
// so its cost follows the block profile of L: how far below the diagonal a panel's nonzero blocks reach.  S couples only
// cameras that share points, but in the order the caller numbered them elimination fills most of L (config 3: L is 26 %
// block-dense for an S that is 1.1 % so).  Reverse Cuthill-McKee keeps the nonzeros of L in a narrow profile, which is what
// a skip of whole row blocks rewards; a minimum-degree order makes L about as sparse but spreads it over many row blocks.
//
// Both orders are scored with the update's own keep rule on the symbolic block structure of L, and RCM is taken only when
// it keeps clearly fewer tiles.  The order permutes the rows and columns of S (schur_final_kernel) and the solution
// (backsub_kernel); a permuted SPD matrix is SPD, so only the rounding of the factorisation changes.
#include "ba_setup.h"
#include "ba_chol_large.cuh"
#include <cstdlib>

namespace bsfm {
namespace ba {

namespace {
struct Graph {
    std::vector<int> ptr, adj, deg;   // free cameras 0 .. nf - 1, neighbours ascending
};

Graph free_graph(int m, int mcon, const uint32_t *keys, int nblocks)
{
    const int nf = m - mcon;
    Graph G;
    G.ptr.assign(nf + 1, 0);
    for (int b = 0; b < nblocks; b++) {
        const int j = (int) (keys[b] / (uint32_t) m), k = (int) (keys[b] % (uint32_t) m);
        if (j != k && j >= mcon && k >= mcon) { G.ptr[j - mcon + 1]++; G.ptr[k - mcon + 1]++; }
    }
    for (int v = 0; v < nf; v++) G.ptr[v + 1] += G.ptr[v];
    G.adj.resize(G.ptr[nf]);
    std::vector<int> fill(G.ptr.begin(), G.ptr.end() - 1);
    for (int b = 0; b < nblocks; b++) {
        const int j = (int) (keys[b] / (uint32_t) m), k = (int) (keys[b] % (uint32_t) m);
        if (j != k && j >= mcon && k >= mcon) { G.adj[fill[j - mcon]++] = k - mcon; G.adj[fill[k - mcon]++] = j - mcon; }
    }
    G.deg.resize(nf);
    for (int v = 0; v < nf; v++) {
        std::sort(G.adj.begin() + G.ptr[v], G.adj.begin() + G.ptr[v + 1]);
        G.deg[v] = G.ptr[v + 1] - G.ptr[v];
    }
    return G;
}

// breadth-first level structure of root's component among the nodes not yet numbered; returns its depth and the last level
int level_structure(const Graph &G, int root, const std::vector<char> &numbered, std::vector<int> &stamp, int tag, std::vector<int> &queue,
                    std::vector<int> &last)
{
    queue.clear(); queue.push_back(root); stamp[root] = tag;
    size_t lo = 0;
    int depth = 0;
    while (true) {
        const size_t hi = queue.size();
        depth++;
        last.assign(queue.begin() + lo, queue.begin() + hi);
        for (size_t q = lo; q < hi; q++)
            for (int e = G.ptr[queue[q]]; e < G.ptr[queue[q] + 1]; e++) {
                const int u = G.adj[e];
                if (!numbered[u] && stamp[u] != tag) { stamp[u] = tag; queue.push_back(u); }
            }
        if (queue.size() == hi) return depth;
        lo = hi;
    }
}

// reverse Cuthill-McKee, component by component in order of their lowest camera: George-Liu pseudo-peripheral start (a
// minimum-degree node of the last level, while that deepens the level structure), neighbours by ascending degree, ties by
// camera index, each component's Cuthill-McKee sequence reversed in place.  order[q] = camera at position q.
std::vector<int> rcm_order(const Graph &G)
{
    const int nf = (int) G.deg.size();
    std::vector<char> numbered(nf, 0);
    std::vector<int> stamp(nf, -1), queue, last, order, nb;
    order.reserve(nf);
    int tag = 0;
    auto lower = [&](int a, int b) { return G.deg[a] != G.deg[b] ? G.deg[a] < G.deg[b] : a < b; };
    for (int start = 0; start < nf; start++) {
        if (numbered[start]) continue;
        int root = start;
        int depth = level_structure(G, root, numbered, stamp, tag++, queue, last);
        while (depth > 1) {
            const int cand = *std::min_element(last.begin(), last.end(), lower);
            const int d = level_structure(G, cand, numbered, stamp, tag++, queue, last);
            root = cand;
            if (d <= depth) break;
            depth = d;
        }
        const size_t c0 = order.size();
        order.push_back(root); numbered[root] = 1;
        for (size_t h = c0; h < order.size(); h++) {
            const int v = order[h];
            nb.clear();
            for (int e = G.ptr[v]; e < G.ptr[v + 1]; e++)
                if (!numbered[G.adj[e]]) nb.push_back(G.adj[e]);
            std::sort(nb.begin(), nb.end(), lower);
            for (int u : nb) { numbered[u] = 1; order.push_back(u); }
        }
        std::reverse(order.begin() + c0, order.end());
    }
    return order;
}

// Tiles chol_solve_large's trailing update keeps for the camera order pos (camera -> position), from the block structure
// of L: column q's structure is S's blocks below the diagonal of camera q plus its elimination-tree children's structures
// (the children are merged as they finish, O(nnz(L))).  A panel's 64-row slab is nonzero when one of its rows belongs to a
// camera coupled in L to a camera of the panel's columns, or to a camera that straddles the panel's end (its own diagonal
// block); the right-hand-side row n always is.  Row block rb (two slabs from the panel's end) is kept when either slab is
// nonzero, and the tiles are the lower triangle of the kept row blocks -- every row block when more than CHOL_MAX_RB.
// Panels stop where the dataflow kernel takes the last <= CHOL_TAIL_MAX columns.  The look-ahead's split of an update into
// two launches keeps the same tiles, so it is not modelled.
int64_t kept_tiles(const Graph &G, const std::vector<int> &pos, int cnp)
{
    const int nf = (int) pos.size(), n = nf * cnp, nrows = n + 1;
    const int npan = (n + LNBO - 1) / LNBO, nslab = (nrows + CHOL_SLAB - 1) / CHOL_SLAB;
    std::vector<int> node(nf);
    for (int v = 0; v < nf; v++) node[pos[v]] = v;
    std::vector<std::vector<int>> str(nf), children(nf);
    std::vector<int> mark(nf, -1);
    std::vector<char> nz((size_t) npan * nslab, 0);
    auto flag_rows = [&](int J, int p) {      // rows of camera position J, below panel p
        const int k1 = std::min(n, (p + 1) * LNBO), r0 = std::max(J * cnp, k1), r1 = (J + 1) * cnp;
        for (int s = r0 / CHOL_SLAB; r0 < r1 && s <= (r1 - 1) / CHOL_SLAB; s++) nz[(size_t) p * nslab + s] = 1;
    };
    for (int q = 0; q < nf; q++) {
        std::vector<int> &s = str[q];
        mark[q] = q;
        const int v = node[q];
        for (int e = G.ptr[v]; e < G.ptr[v + 1]; e++) {
            const int r = pos[G.adj[e]];
            if (r > q && mark[r] != q) { mark[r] = q; s.push_back(r); }
        }
        for (int c : children[q]) {
            for (int r : str[c]) if (mark[r] != q) { mark[r] = q; s.push_back(r); }
            std::vector<int>().swap(str[c]);
        }
        if (!s.empty()) children[*std::min_element(s.begin(), s.end())].push_back(q);
        const int p0 = q * cnp / LNBO, p1 = ((q + 1) * cnp - 1) / LNBO;   // the panels camera q's columns lie in
        for (int p = p0; p <= p1; p++) {
            for (int r : s) flag_rows(r, p);
            flag_rows(q, p);      // nonzero below k1 only when the camera straddles the panel's end
        }
    }
    int64_t tiles = 0;
    std::vector<int> kept;
    for (int p = 0; p < npan; p++) {
        const int k0 = p * LNBO, k1 = std::min(n, k0 + LNBO);
        if (k0 > 0 && n - k0 <= CHOL_TAIL_MAX && n - k0 > 2 * LNB) break;      // the dataflow tail
        if (k1 >= n) break;
        const char *f = nz.data() + (size_t) p * nslab;
        const int nrb = (nrows - k1 + CHOL_TILE - 1) / CHOL_TILE, ncb = (n - k1 + CHOL_TILE - 1) / CHOL_TILE;
        const int s0 = k1 / CHOL_SLAB, send = (nrows - 1) / CHOL_SLAB;      // slabs of the rows below the panel (k1 is 64-aligned)
        kept.clear();
        for (int rb = 0; rb < nrb; rb++) {
            const int s = s0 + 2 * rb;
            const bool keep = nrb > CHOL_MAX_RB || s == send || s + 1 == send || f[s] || (s + 1 <= send && f[s + 1]);
            if (keep) kept.push_back(rb);
        }
        for (size_t j = 0; j < kept.size() && kept[j] < ncb; j++) tiles += (int64_t) (kept.size() - j);
    }
    return tiles;
}
}  // namespace

int camera_order(int m, int mcon, int cnp, const uint32_t *keys, int nblocks, std::vector<int> &pos, int64_t scores[2])
{
    const int nf = m - mcon;
    pos.resize(nf);
    for (int v = 0; v < nf; v++) pos[v] = v;
    scores[0] = scores[1] = 0;
    if ((int64_t) nf * cnp <= CHOL_LARGE_MIN) return 0;      // the small paths skip nothing: the order cannot pay
    const Graph G = free_graph(m, mcon, keys, nblocks);
    const std::vector<int> order = rcm_order(G);
    std::vector<int> rpos(nf);
    for (int q = 0; q < nf; q++) rpos[order[q]] = q;
    scores[0] = kept_tiles(G, pos, cnp);
    scores[1] = kept_tiles(G, rpos, cnp);
    if (4 * scores[1] > 3 * scores[0]) return 0;      // RCM only when it keeps at most three quarters of the tiles
    pos.swap(rpos);
    return 1;
}

// first nonzero column of every row of S in the camera order pos: row block q of camera position q starts at
// cnp x min(position of q's neighbours and of q itself)
static std::vector<int> band_first_cols(int m, int mcon, int cnp, const uint32_t *keys, int nblocks, const std::vector<int> &pos)
{
    const int nf = m - mcon;
    std::vector<int> lo(pos);      // lo[v]: lowest position among camera v and its neighbours
    for (int b = 0; b < nblocks; b++) {
        const int j = (int) (keys[b] / (uint32_t) m), k = (int) (keys[b] % (uint32_t) m);
        if (j < mcon || k < mcon) continue;
        lo[j - mcon] = std::min(lo[j - mcon], pos[k - mcon]);
        lo[k - mcon] = std::min(lo[k - mcon], pos[j - mcon]);
    }
    std::vector<int> first((size_t) nf * cnp);
    for (int v = 0; v < nf; v++)
        for (int r = 0; r < cnp; r++) first[(size_t) pos[v] * cnp + r] = lo[v] * cnp;
    return first;
}

// The tiles with an update step, by interval colouring in order of first step (ties: ascending tile index): each takes the
// lowest colour whose previous tile finished before it starts, so the colours used are the largest live set and every
// colour's tiles follow each other in increasing step.  Colour c is slot c / workers of worker c % workers.
void chol_band_plan(int n, const int *first_col, int max_workers, CholBandPlan &plan)
{
    plan = CholBandPlan();
    const int nbk = (n + LNB - 1) / LNB;
    plan.n = n; plan.nbk = nbk;
    plan.env.assign(nbk + 1, 0);
    for (int rb = 0; rb < nbk; rb++) {
        int e = rb * LNB;
        for (int i = rb * LNB; i < std::min(n, (rb + 1) * LNB); i++) e = std::min(e, std::max(0, std::min(first_col[i], i)));
        plan.env[rb] = e / LNB;
    }
    plan.toff.assign(nbk + 2, 0);
    for (int rb = 0; rb <= nbk; rb++) plan.toff[rb + 1] = plan.toff[rb] + (rb == nbk ? nbk : rb - plan.env[rb] + 1);
    plan.ntile = plan.toff[nbk + 1];
    struct Live { int kf, kl, rb, cb; };
    std::vector<Live> live;
    for (int rb = 0; rb <= nbk; rb++)
        for (int cb = plan.env[rb]; cb < std::min(rb + 1, nbk); cb++) {
            const int kf = std::max(plan.env[rb], plan.env[cb]), kl = (rb == cb) ? cb - 2 : cb - 1;
            if (kf <= kl) live.push_back({kf, kl, rb, cb});
        }
    std::vector<int> starts(nbk + 1, 0), ends(nbk + 1, 0);
    for (const Live &t : live) { starts[t.kf]++; ends[t.kl]++; }
    for (int k = 0, cur = 0; k < nbk; k++) { cur += starts[k]; plan.max_live = std::max(plan.max_live, cur); cur -= ends[k]; }
    plan.workers = std::max(1, std::min(max_workers, plan.max_live));
    plan.fits = n > CHOL_BAND_MIN_N && n <= CHOL_BAND_MAX_N && max_workers >= 1 && plan.max_live <= 2 * plan.workers &&
                (size_t) plan.ntile <= chol_band_capacity_tiles(n);
    if (!plan.fits) return;      // a wide envelope is refused before the colouring, whose cost grows with its width
    // intervals in order of start: the lowest free colour uses exactly max_live colours
    std::stable_sort(live.begin(), live.end(), [](const Live &a, const Live &b) { return a.kf < b.kf; });
    std::vector<int> colour_end, colour(live.size());      // last step of every colour's latest tile
    for (size_t t = 0; t < live.size(); t++) {
        int c = 0;
        while (c < (int) colour_end.size() && colour_end[c] >= live[t].kf) c++;
        if (c == (int) colour_end.size()) colour_end.push_back(0);
        colour_end[c] = live[t].kl;
        colour[t] = c;
    }
    const int W = plan.workers;
    plan.sptr.assign(2 * W + 1, 0);
    for (size_t t = 0; t < live.size(); t++) plan.sptr[2 * (colour[t] % W) + colour[t] / W + 1]++;
    for (int s = 0; s < 2 * W; s++) plan.sptr[s + 1] += plan.sptr[s];
    plan.sched.resize(live.size());
    std::vector<int> fill(plan.sptr.begin(), plan.sptr.end() - 1);
    for (size_t t = 0; t < live.size(); t++) plan.sched[fill[2 * (colour[t] % W) + colour[t] / W]++] = live[t].rb << 16 | live[t].cb;
}

int apply_camera_order(Problem &P, int cnp, cudaStream_t st, DeviceArena &D, CholBand &band)
{
    static const bool on = []() { const char *e = getenv("BSFM_BA_CAMERA_ORDER"); return !(e && e[0] == '0'); }();
    P.cam_pos = nullptr;
    band = CholBand();
    const int nf = P.m - P.mcon;
    const int64_t nsys = (int64_t) nf * cnp;
    if (nsys <= CHOL_LARGE_MIN || P.nblocks <= 0 || (!on && nsys <= CHOL_BAND_MIN_N)) return BSFM_OK;
    std::vector<uint32_t> keys(P.nblocks);
    BSFM_CUDA_TRY(cudaMemcpyAsync(keys.data(), P.blk_key, keys.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<int> pos(nf);
    for (int v = 0; v < nf; v++) pos[v] = v;
    int64_t scores[2];
    const bool rcm = on && camera_order(P.m, P.mcon, cnp, keys.data(), P.nblocks, pos, scores);
    if (rcm) {
        int *d_pos;
        TRY(D.upload(&d_pos, pos.data(), pos.size()));      // pageable source: the copy is staged before it returns
        P.cam_pos = d_pos;
    }
    // the envelope of S in the order it is factored in; its plan, when it fits, replaces the panel path
    if (nsys <= CHOL_BAND_MIN_N) return BSFM_OK;
    int dev = 0, sms = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    BSFM_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const std::vector<int> first = band_first_cols(P.m, P.mcon, cnp, keys.data(), P.nblocks, pos);
    CholBandPlan plan;
    chol_band_plan(nf * cnp, first.data(), sms - 1, plan);
    if (!plan.fits) return BSFM_OK;
    return upload_band_plan(plan, D, band);
}

int upload_band_plan(const CholBandPlan &plan, DeviceArena &D, CholBand &band)
{
    int *env, *toff, *sptr, *sched;
    TRY(D.upload(&env, plan.env.data(), plan.env.size()));
    TRY(D.upload(&toff, plan.toff.data(), plan.toff.size()));
    TRY(D.upload(&sptr, plan.sptr.data(), plan.sptr.size()));
    TRY(D.upload(&sched, plan.sched.data(), plan.sched.size()));
    band.env = env; band.toff = toff; band.sptr = sptr; band.sched = sched;
    band.ntile = plan.ntile; band.workers = plan.workers;
    return BSFM_OK;
}

}  // namespace ba
}  // namespace bsfm

extern "C" int bsfm_ba_camera_order(int m, int mcon, int cnp, const uint32_t *blk_key, int nblocks, int32_t *cam_pos, int64_t scores[2])
{
    using namespace bsfm;
    clear_error();
    if (m <= 0 || mcon < 0 || mcon >= m || cnp <= 0 || nblocks < 0 || (nblocks > 0 && !blk_key) || !cam_pos || !scores) {
        set_error("bsfm_ba_camera_order: bad arguments");
        return BSFM_ERR_ARG;
    }
    for (int b = 0; b < nblocks; b++) {
        const uint32_t j = blk_key[b] / (uint32_t) m, k = blk_key[b] % (uint32_t) m;
        if (j > k || k >= (uint32_t) m) { set_error("bsfm_ba_camera_order: block key %u is not j * m + k with j <= k < m", blk_key[b]); return BSFM_ERR_ARG; }
    }
    std::vector<int> pos;
    const int rcm = ba::camera_order(m, mcon, cnp, blk_key, nblocks, pos, scores);
    std::copy(pos.begin(), pos.end(), cam_pos);
    return rcm;
}

extern "C" int bsfm_ba_chol_band_plan(int n, const int32_t *first_col, int workers, int32_t *env, int64_t out[3])
{
    using namespace bsfm;
    clear_error();
    if (n <= 0 || n > (1 << 20) || !first_col || workers < 1 || !out) { set_error("bsfm_ba_chol_band_plan: bad arguments"); return BSFM_ERR_ARG; }
    for (int i = 0; i < n; i++)
        if (first_col[i] < 0 || first_col[i] > i) { set_error("bsfm_ba_chol_band_plan: first_col[%d] = %d is not in [0, %d]", i, first_col[i], i); return BSFM_ERR_ARG; }
    ba::CholBandPlan plan;
    ba::chol_band_plan(n, first_col, workers, plan);
    if (env) std::copy(plan.env.begin(), plan.env.end(), env);
    out[0] = plan.ntile; out[1] = plan.max_live; out[2] = plan.fits ? plan.workers : 0;
    return plan.fits ? 1 : 0;
}
