/* oracle/match_oracle.c -- TEST INFRASTRUCTURE ONLY (CPU restatement; never shipped, never timed
 * as the product).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
 * load this.
 *
 * Restates the MATCH hot path of snavely/bundler_sfm in exact mode:
 *   MatchKeys(n1,k1,tree2,ratio,max_pts_visit=0)      src/keys2a.cpp:347-372
 *   distance arithmetic  t=(int)q-(int)p; dist+=t*t   lib/ann_1.1_char/src/kd_pr_search.cpp:194-209
 *   2-best queue, INT_MAX / -1 when fewer than k pts   lib/ann_1.1_char/src/pr_queue_k.h:69-119,
 *                                                      include/ANN/ANN.h:202 (ANN_DIST_INF=INT_MAX)
 *   ratio test (double)d0 < ratio*ratio*(double)d1    src/keys2a.cpp:362
 *   pair loop + ">= 16 matches" table writer           src/KeyMatchFull.cpp:105-151
 *
 * Pinning: validated bit-for-bit against oracle/_ref/libref_match.so (the reference compiled
 * from /root/reference, exact mode max_pts_visit=0) by tests/test_oracle_match.py, and against
 * the committed vectors in tests/golden/match_*.npz which that reference produced.
 *
 * Tie note: when two database keys tie for the best distance, d0==d1.  The keys2a test cannot
 * pass then for ratio<=1 (KeyMatchFull hard-codes 0.6), so which tied key wins is unobservable.
 * The keys.cpp test sqrt(d0/d1) <= ratio passes it at ratio 1.0, which the symmetric pass of
 * bundler --add_images uses (Bundle.cpp:3817-3820), so there the tied key is part of the output.
 * This port returns the smallest caller index among the tied keys (first seen), and so does every
 * GPU kernel.  The unmodified kd-tree returns the first tied key it visits, which can be another
 * (tests/golden/match_ties_golden.npz records where).
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define DESC_DIM 128

/* squared L2 in int32, as kd_pr_search.cpp:200-209 without the early exit (same value) */
static int sqdist128(const unsigned char *q, const unsigned char *p)
{
    int dist = 0, d;
    for (d = 0; d < DESC_DIM; d++) {
        int t = (int) q[d] - (int) p[d];
        dist += t * t;
    }
    return dist;
}

/* exact 2-NN of one query against n2 database keys: pr_queue_k.h insertion semantics
 * (strict '>' shift => first-seen wins ties) */
void oracle_top2(const unsigned char *q, const unsigned char *k2, int n2,
                 int *d0, int *d1, int *i0, int *i1)
{
    int b0 = INT_MAX, b1 = INT_MAX, j0 = -1, j1 = -1, j;
    for (j = 0; j < n2; j++) {
        int d = sqdist128(q, k2 + (size_t) DESC_DIM * j);
        if (d < b0)      { b1 = b0; j1 = j0; b0 = d; j0 = j; }
        else if (d < b1) { b1 = d;  j1 = j; }
    }
    *d0 = b0; *d1 = b1; *i0 = j0; *i1 = j1;
}

/* keys2a.cpp:347-372 in exact mode.  out_pairs gets (idx1, idx2) for the first `cap` matches;
 * the return value is the total number of matches (may exceed cap). */
int oracle_match_pair(const unsigned char *k1, int n1, const unsigned char *k2, int n2,
                      double ratio, int32_t *out_pairs, int cap)
{
    int cnt = 0, i;
    if (n1 <= 0 || n2 <= 0) return 0;
    for (i = 0; i < n1; i++) {
        int d0, d1, i0, i1;
        oracle_top2(k1 + (size_t) DESC_DIM * i, k2, n2, &d0, &d1, &i0, &i1);
        if (((double) d0) < ratio * ratio * ((double) d1)) {   /* keys2a.cpp:362 */
            if (cnt < cap) { out_pairs[2 * cnt] = i; out_pairs[2 * cnt + 1] = i0; }
            cnt++;
        }
    }
    return cnt;
}

/* The in-bundler matcher, src/keys.cpp:961-1057 (MatchKeysExhaustive; MatchKeys :717-810 is the same loop on an approximate
 * search): accept iff sqrt((double) d0 / (double) d1) <= ratio (:786, :1029).  mode 0 = the keys2a test above.
 * (`registered` is applied by the caller: it only selects which keys of image 2 form the database.) */
int oracle_match_pair_test(const unsigned char *k1, int n1, const unsigned char *k2, int n2,
                           double ratio, int mode, int32_t *out_pairs, int cap)
{
    int cnt = 0, i;
    if (mode == 0) return oracle_match_pair(k1, n1, k2, n2, ratio, out_pairs, cap);
    if (n1 <= 0 || n2 <= 0) return 0;
    for (i = 0; i < n1; i++) {
        int d0, d1, i0, i1;
        oracle_top2(k1 + (size_t) DESC_DIM * i, k2, n2, &d0, &d1, &i0, &i1);
        if (sqrt(((double) d0) / ((double) d1)) <= ratio) {
            if (cnt < cap) { out_pairs[2 * cnt] = i; out_pairs[2 * cnt + 1] = i0; }
            cnt++;
        }
    }
    return cnt;
}

/* also expose the raw (d0,d1,i0) per query for kernel-level unit tests */
void oracle_top2_all(const unsigned char *k1, int n1, const unsigned char *k2, int n2,
                     int32_t *d0, int32_t *d1, int32_t *i0)
{
    int i;
    for (i = 0; i < n1; i++) {
        int a, b, c, d;
        oracle_top2(k1 + (size_t) DESC_DIM * i, k2, n2, &a, &b, &c, &d);
        d0[i] = a; d1[i] = b; i0[i] = c;
    }
}

/* KeyMatchFull.cpp:105-151: for i ascending, for j in [max(i-window,0), i): match j -> i.
 * keys = concatenation of all images' descriptors, key_off[i] = first key of image i (N+1 entries).
 * Writes the text match table into buf (if non-NULL, up to buf_cap bytes) and returns the number
 * of bytes the full table needs.  pair_counts (optional, N*N ints) receives every pair's match
 * count at [i*N+j] (also pairs below the 16-match write threshold). */
long oracle_match_all_pairs(const unsigned char *keys, const int64_t *key_off, int N,
                            int window_radius, double ratio, int min_matches,
                            char *buf, long buf_cap, int32_t *pair_counts)
{
    long pos = 0;
    int i, j, k;
    int maxk = 0;
    int32_t *tmp;
    for (i = 0; i < N; i++) {
        int n = (int) (key_off[i + 1] - key_off[i]);
        if (n > maxk) maxk = n;
    }
    tmp = (int32_t *) malloc(sizeof(int32_t) * 2 * (size_t) (maxk > 0 ? maxk : 1));
    for (i = 0; i < N; i++) {
        int ni = (int) (key_off[i + 1] - key_off[i]);
        int start_idx = 0;
        if (ni == 0) continue;                                  /* :106-107 */
        if (window_radius > 0) start_idx = (i - window_radius > 0) ? i - window_radius : 0;  /* :116-119 */
        for (j = start_idx; j < i; j++) {
            int nj = (int) (key_off[j + 1] - key_off[j]);
            int cnt;
            if (nj == 0) continue;                              /* :122-123 */
            cnt = oracle_match_pair(keys + DESC_DIM * key_off[j], nj,
                                    keys + DESC_DIM * key_off[i], ni, ratio, tmp, maxk);
            if (pair_counts) pair_counts[(size_t) i * N + j] = cnt;
            if (cnt >= min_matches) {                           /* :131 (16) */
                char line[64];
                int len = snprintf(line, sizeof line, "%d %d\n%d\n", j, i, cnt);
                if (buf && pos + len <= buf_cap) memcpy(buf + pos, line, len);
                pos += len;
                for (k = 0; k < cnt; k++) {
                    len = snprintf(line, sizeof line, "%d %d\n", tmp[2 * k], tmp[2 * k + 1]);
                    if (buf && pos + len <= buf_cap) memcpy(buf + pos, line, len);
                    pos += len;
                }
            }
        }
    }
    free(tmp);
    return pos;
}
