/* bsfm_b200.h -- C ABI of libbsfm_b200.so, the H100-native (sm_90a) drop-in for the two
 * data-parallel hot paths of snavely/bundler_sfm.  Plain pointers and sizes only; no torch types.
 * Every entry point cites the reference interface (file:line under /root/reference) it replaces.
 *
 *   MATCH  : all-pairs 128-D uint8 SIFT 2-NN + ratio test  (src/keys2a.cpp, src/KeyMatchFull.cpp)
 *   BA     : sparse Levenberg-Marquardt bundle adjustment   (lib/sfm-driver/sfm.c, lib/sba-1.5)
 *
 * Error convention: functions returning int/int64 return a negative value on failure and store a
 * message retrievable with bsfm_last_error().  There is NO CPU fallback: without a CUDA device (or
 * without the sm_90a kernels) every compute entry point fails loudly.
 */
#ifndef BSFM_B200_H
#define BSFM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BSFM_OK              0
#define BSFM_ERR_CUDA       -2   /* CUDA runtime / launch error (message has the detail)        */
#define BSFM_ERR_ARG        -3   /* invalid argument                                            */
#define BSFM_ERR_CAPACITY   -4   /* caller-provided output buffer too small (needed size known)  */
#define BSFM_ERR_NO_DEVICE  -5   /* no usable sm_90 GPU                                         */
#define BSFM_ERR_UNSUPPORTED -6  /* reference feature outside the GPU path (see INTEGRATION.md)  */

/* last error message of the calling thread's most recent failing call ("" if none) */
const char *bsfm_last_error(void);
/* library version string, e.g. "bsfm_b200 0.1 (sm_90a)" */
const char *bsfm_version(void);
/* number of kernels launched by this process through the library so far (bench `gpu_launches`) */
int64_t bsfm_kernel_launches(void);
/* select the CUDA device used by subsequent calls of this thread's process (default: current) */
int bsfm_set_device(int device);
/* Measured int8 tensor-pipe ceiling of the current device in TOP/s (2 ops per multiply-add): a plain wgmma u8 loop,
 * two warpgroups per SM, M = 64, N = n_tile (128 or 256), operands resident in shared memory, no loads, no epilogue (csrc/tc_peak.cu).
 * bench.py uses it as the denominator of the tensor rooflines (SURVEY.md 8d).  < 0 on error.                        */
double bsfm_measure_int8_peak(int n_tile, int iters);
/* Measured fp64 issue interval of the current device: SM cycles per warp instruction per SM sub-partition with `warps` resident
 * warps of one CTA; mode 0 = vector DFMA (8 independent chains per thread), mode 1 = DMMA m8n8k4 (4 independent accumulators),
 * mode 2 = DMMA m16n8k8 (4 independent accumulators; the shape of the large Cholesky's trailing update, 2048 fp64 FLOP per
 * instruction, so 2048 * 4 / cycles is the SM's fp64 tensor rate in FLOP per clock).  The numbers behind DESIGN.md's notes
 * on the Cholesky (csrc/tc_peak.cu).  < 0 on error.                                                              */
double bsfm_measure_fp64_issue_cycles(int mode, int warps, int iters);
/* number of CUDA devices visible to this process (0 when there is none) */
int bsfm_device_count(void);

/* ------------------------------------------------------------------------------------------------
 * MATCH
 * ---------------------------------------------------------------------------------------------- */

/* kernel selector for the matcher (env BSFM_MATCH_KERNEL overrides the default):
 *   0 = wgmma u8 tensor-core kernel (TMA bulk loads, register accumulators)   [default]
 *   1 = DP4A CUDA-core kernel (independent second implementation used to cross-check; not a fallback)
 * further switches of kernel 0 (all variants return identical results, DESIGN.md 3.2):
 *   BSFM_MATCH_EPILOGUE=0  exact chunk-minimum epilogue instead of the bound epilogue (automatic for databases with
 *                          an image of more than 8192 padded rows)
 *   BSFM_MATCH_QUAD=1      four register accumulators of 64 columns per database tile instead of two of 128
 *   BSFM_MATCH_PAIR=1      CTA-pair kernel (clusters of two CTAs, each loads half of every database tile and multicasts
 *                          it to both with TMA)                                                                      */
#define BSFM_MATCH_KERNEL_TC    0
#define BSFM_MATCH_KERNEL_DP4A  1

/* Replaces  std::vector<KeypointMatch> MatchKeys(int num_keys1, unsigned char *k1,
 *                                               int num_keys2, unsigned char *k2,
 *                                               double ratio, int max_pts_visit)
 *           src/keys2a.h:99-102, src/keys2a.cpp:375-424   (and the tree overload :347-372 via the
 *           C++ shim in shim/keys2a_b200.cpp).
 * For every query i in k1 finds the two nearest keys in k2 under squared L2 (int32) and emits
 * (i, nn0) iff (double)d0 < ratio*ratio*(double)d1 (keys2a.cpp:362), ascending in i.
 * The search is EXACT (== the reference with max_pts_visit = 0; the reference default of 200 is an
 * approximation, SURVEY.md F2).  k1: n1 x 128 bytes, k2: n2 x 128 bytes, host memory.
 * out_pairs: cap x 2 int32 (idx1, idx2).  Returns the number of matches (>=0); if it exceeds cap,
 * only the first cap are written and the full count is still returned.                       */
int bsfm_match_pair(const uint8_t *k1, int n1, const uint8_t *k2, int n2, double ratio,
                    int32_t *out_pairs, int cap);
/* The same 2-NN search with a selectable acceptance test:
 *   BSFM_RATIO_TEST_KEYS2A  (double) d0 < ratio^2 (double) d1           MatchKeys of src/keys2a.cpp:362, :412 (KeyMatchFull)
 *   BSFM_RATIO_TEST_KEYS    sqrt((double) d0 / (double) d1) <= ratio    MatchKeys / MatchKeysExhaustive of src/keys.cpp:786, :1029
 *                           (bundler --add_images, src/Bundle.cpp:3812-3820; d1 = INT_MAX when image 2 has one key)
 * Exact search, i.e. keys.cpp's MatchKeysExhaustive (the stock MatchKeys there caps the kd-tree search at 200 visits).
 * For ratio >= 1 the partner reported for a query whose two nearest keys are EXACTLY equidistant is the one with the
 * smaller index (the reference reports whichever its kd-tree meets first).                                             */
#define BSFM_RATIO_TEST_KEYS2A 0
#define BSFM_RATIO_TEST_KEYS   1
int bsfm_match_pair_test(const uint8_t *k1, int n1, const uint8_t *k2, int n2, double ratio, int ratio_test,
                         int32_t *out_pairs, int cap);
/* bsfm_match_pair keeps the prepared device image of every key buffer it has seen (keyed by key count and a 64-bit hash
 * of the contents; the unmodified KeyMatchFull main passes the same buffers for every pair, KeyMatchFull.cpp:105-151),
 * least recently used images are dropped beyond 8 GB.  This releases them all.                                       */
void bsfm_match_pair_cache_clear(void);

/* Device-resident key database for the KeyMatchFull all-pairs loop (src/KeyMatchFull.cpp:93-151).
 * keys  : concatenation of all images' descriptors (sum n_i x 128 bytes), HOST memory
 * key_off: N+1 prefix offsets in keys (units of descriptors)
 * Uploads once, computes squared norms, sorts the keys of every image by norm and writes the padded,
 * 128B-swizzled tile layout the tensor-core kernel streams with TMA bulk copies (DESIGN.md 3.1);
 * results are always reported in the caller's key order.                                      */
typedef struct bsfm_keydb bsfm_keydb;
bsfm_keydb *bsfm_keydb_create(const uint8_t *keys, const int64_t *key_off, int num_images);
/* same, but `keys_dev` already lives in device memory (bench `value` leg; torch data_ptr()) */
bsfm_keydb *bsfm_keydb_create_dev(const uint8_t *keys_dev, const int64_t *key_off, int num_images);
void bsfm_keydb_destroy(bsfm_keydb *db);

/* Number of ordered image pairs (j < i, j >= i - window_radius if window_radius > 0) the
 * KeyMatchFull loop visits (KeyMatchFull.cpp:105-121), in its order: i ascending, j ascending.
 * Pairs with an empty image are included (they produce 0 matches).                           */
int64_t bsfm_match_num_pairs(int num_images, int window_radius);

/* Runs the pair loop of KeyMatchFull.cpp:105-151 for the database images i in [img_begin, img_end)
 * (all j < i inside the window), i.e. one contiguous shard of the pair list -- the unit of
 * multi-GPU sharding.  Results stay on the device inside `db` until fetched.
 * Returns the total number of matches found in the shard (>=0) or a negative error.          */
int64_t bsfm_match_run(bsfm_keydb *db, int img_begin, int img_end, int window_radius, double ratio);

/* Copies the result of the last bsfm_match_run to host memory.
 * pair_counts : one int32 per pair of the shard, KeyMatchFull order
 * matches     : total x 2 int32 (idx_in_j, idx_in_i), grouped by pair in the same order, ascending
 *               idx_in_j inside a pair (keys2a.cpp:356-365)
 * Returns BSFM_OK or BSFM_ERR_CAPACITY.                                                       */
int bsfm_match_fetch(bsfm_keydb *db, int32_t *pair_counts, int64_t pair_cap,
                     int32_t *matches, int64_t match_cap);
/* device pointers of the same two arrays (valid until the next run/destroy) for an NCCL
 * all-gather straight from HBM; *num_pairs / *num_matches receive the element counts          */
int bsfm_match_result_dev(bsfm_keydb *db, const int32_t **pair_counts_dev, int64_t *num_pairs,
                          const int32_t **matches_dev, int64_t *num_matches);
/* device-to-device copy of the same two arrays into caller-owned DEVICE buffers (e.g. torch tensors
 * that then feed torch.distributed all_gather over NCCL)                                        */
int bsfm_match_copy_result_dev(bsfm_keydb *db, int32_t *pair_counts_dst_dev, int32_t *matches_dst_dev);
/* number of pairs in the shard of the last run */
int64_t bsfm_match_shard_pairs(bsfm_keydb *db);
/* timing of the last bsfm_match_run measured with CUDA events on the launching stream:
 * ms[0] = search kernel(s), ms[1] = verify+sort+finalize, ms[2] = whole run; launches = kernels  */
int bsfm_match_last_timing(bsfm_keydb *db, float ms[3], int *launches);

/* One-call host API: KeyMatchFull's loop over host buffers (upload + run + fetch).
 * Returns total matches or negative error; BSFM_ERR_CAPACITY if match_cap too small.          */
int64_t bsfm_match_all_pairs(const uint8_t *keys, const int64_t *key_off, int num_images,
                             int window_radius, double ratio,
                             int32_t *pair_counts, int64_t pair_cap,
                             int32_t *matches, int64_t match_cap);

/* ------------------------------------------------------------------------------------------------
 * BA  (declared in bsfm_b200_ba.h; kept separate because it mirrors the reference structs)
 * ---------------------------------------------------------------------------------------------- */

/* ---- multi-GPU (SURVEY.md 8e): the KeyMatchFull pair loop (src/KeyMatchFull.cpp:105-151) sharded by database image, one
 * communicator rank per GPU, NCCL over NVLink.  Works with one process per GPU (the id travels through whatever launcher
 * the caller has: bench.py broadcasts it with torch.distributed) and with several host threads in one process.
 * NCCL (libnccl.so.2) is bound at run time; without it these entry points return BSFM_ERR_UNSUPPORTED.               */
typedef struct bsfm_comm bsfm_comm;
#define BSFM_COMM_ID_BYTES 128
int bsfm_comm_unique_id(unsigned char id[BSFM_COMM_ID_BYTES]);                                /* rank 0: ncclGetUniqueId */
bsfm_comm *bsfm_comm_create(const unsigned char id[BSFM_COMM_ID_BYTES], int rank, int world_size);   /* on the CURRENT device */
void bsfm_comm_destroy(bsfm_comm *comm);
/* cooperative bsfm_keydb_create: rank r uploads and prepares (norm sort + swizzle) only its 1/world share of the images;
 * the prepared rows are exchanged with one in-place ncclAllGather per array; every rank ends with the whole database.
 * Collective: every rank of `comm` must call it with the same arguments.                                            */
bsfm_keydb *bsfm_keydb_create_sharded(bsfm_comm *comm, const uint8_t *keys, const int64_t *key_off, int num_images);
/* contiguous database-image range of `rank`: equal shares of the work n_i * sum_{j in window} n_j                    */
int bsfm_match_shard_range(const int64_t *key_off, int num_images, int window_radius, int world_size, int rank, int *img_begin, int *img_end);
/* all-gather of the ranks' tables after each ran bsfm_match_run on its range (ranges in rank order): count all-gather,
 * then one grouped broadcast per rank into its offset of the concatenated table (== the KeyMatchFull order).  Collective.
 * Returns the total number of matches; the table stays in device memory of every rank.                               */
int64_t bsfm_match_allgather(bsfm_comm *comm, bsfm_keydb *db);
/* gathered table -> host or device buffers (*num_pairs / *num_matches = sizes of the whole table; null buffers: sizes only) */
int bsfm_match_gathered_fetch(bsfm_keydb *db, int64_t *num_pairs, int64_t *num_matches, int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap);
/* bsfm_match_all_pairs on `ngpus` devices of this process (one host thread per GPU; devices == NULL: 0 .. ngpus-1):
 * the export SURVEY.md 8b names for the multi-GPU KeyMatchFull.  Same outputs as bsfm_match_all_pairs.               */
int64_t bsfm_match_all_pairs_multi(const uint8_t *keys, const int64_t *key_off, int num_images, int window_radius, double ratio,
                                   int ngpus, const int *devices, int32_t *pair_counts, int64_t pair_cap, int32_t *matches, int64_t match_cap);

#ifdef __cplusplus
}
#endif
#endif /* BSFM_B200_H */
