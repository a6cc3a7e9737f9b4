/* dsk.h -- C-ABI of libdsk_b200.so: the H100 (sm_90a) MinHash / LSH signature engine.
 *
 * The reference (ekzhu/datasketch 1.10.0) is pure Python and exposes NO plugin /
 * FFI interface; its only backend seam is the `gpu_mode` switch inside
 * MinHash.update_batch (datasketch/minhash.py:117, :270-291).  This header is the
 * boundary a maintainer would bind with ctypes to replace that seam and the
 * Python loops around it (see INTEGRATION.md for the stub).  Each entry point
 * cites the reference code it replaces.
 *
 * Conventions
 *   - plain C types only; no torch / CUDA types in signatures (streams are void*,
 *     i.e. a cudaStream_t / CUstream value; NULL = the legacy default stream).
 *   - "d_" parameters are DEVICE pointers owned by the caller (e.g. torch tensors'
 *     data_ptr()); "h_" parameters are HOST pointers.
 *   - device entry points are stream-ordered and asynchronous; return 0 when the
 *     work was enqueued, non-zero DSK_ERR_* otherwise; dsk_last_error() returns a
 *     thread-local message for the last failure on the calling thread.
 *   - integer results are bit-exact with the reference's numpy uint64 path.
 */
#ifndef DSK_H_
#define DSK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSK_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define DSK_API __attribute__((visibility("default")))
#else
#define DSK_API
#endif

enum {
    DSK_OK = 0,
    DSK_ERR_INVALID = 1,   /* bad argument (maps to ValueError in the Python host layer) */
    DSK_ERR_CUDA = 2,      /* CUDA runtime error (maps to RuntimeError) */
    DSK_ERR_NO_DEVICE = 3, /* no sm_90 device: there is NO CPU fallback (RuntimeError) */
    DSK_ERR_ALIGN = 4,     /* pointer alignment contract violated */
    DSK_ERR_NOMEM = 5
};

/* kernel selection for dsk_minhash_bulk (flags) */
enum {
    DSK_KERNEL_AUTO = 0,     /* = TWO_PHASE */
    DSK_KERNEL_TWO_PHASE = 1,/* the two-phase signature kernel; bit-exact for ANY permutation and u32 / u64 tokens: the default
                                variant needs 32-bit tokens and n_unsafe == 0, otherwise a general variant runs that
                                takes the conditional subtract of `% (2^61-1)` in its exact stage (window 8 instead of 7) */
    DSK_KERNEL_DIRECT = 2,   /* r = lo32(x) + top3(x) per (token, perm), no candidate filtering; DSK_ERR_INVALID unless
                                the tokens are 32-bit and n_unsafe == 0 */
    DSK_KERNEL_EXACT = 3     /* full 64-bit `% (2^61-1)` per evaluation; any permutation, u32/u64 tokens (round 1's kernel) */
};

DSK_API int dsk_version(void);
DSK_API const char *dsk_last_error(void);

/* Number of usable CUDA devices; *sm_count / *cc receive properties of `device`.
 * Replaces datasketch/minhash.py:38-48 (_gpu_available). */
DSK_API int dsk_device_count(void);
DSK_API int dsk_device_info(int device, int *sm_count, int *cc_major, int *cc_minor, size_t *total_mem);

/* ---- permutation handle -------------------------------------------------------
 * Uploads the (a, b) parameters of MinHash._init_permutations
 * (datasketch/minhash.py:170-184; generated on the HOST with numpy, never on
 * device) and analyses them once: `n_unsafe` = number of permutations for which
 * some 32-bit token value h makes ((a*h+b) mod 2^64) fall in the 36-value set
 * where `% (2^61-1)` needs its conditional subtract.  n_unsafe == 0 (true for every seed-generated
 * set tested) selects the two-phase kernel's default variant and allows DSK_KERNEL_DIRECT; otherwise the
 * two-phase kernel's general variant runs (same speed class, still bit-exact).
 * Replaces minhash.py:160-165 (_ensure_gpu_caches). */
typedef struct dsk_perm dsk_perm;
DSK_API int dsk_perm_create(const uint64_t *h_a, const uint64_t *h_b, int num_perm, int device, dsk_perm **out);
DSK_API int dsk_perm_info(const dsk_perm *p, int *num_perm, int *n_unsafe, int *device);
DSK_API void dsk_perm_destroy(dsk_perm *p);
/* Host-only analysis (no device needed): out_unsafe[i] = 1 iff permutation i can reach the
 * conditional-subtract set with some token h < 2^32.  Returns the number of unsafe ones. */
DSK_API int dsk_perm_analyze(const uint64_t *h_a, const uint64_t *h_b, int num_perm, uint8_t *out_unsafe);

/* ---- bulk signature build -------------------------------------------------------
 * Replaces MinHash.update_batch's hot loop (datasketch/minhash.py:294-297 CPU,
 * :281-291 CuPy) batched over documents as in MinHash.bulk / generator
 * (:464-522): for document i with token hashes tokens[offsets[i]:offsets[i+1]],
 *   out[i][k] = min(init[i][k], min_t (((a_k*h_t + b_k) mod 2^64) % (2^61-1)) & 0xFFFFFFFF)
 * d_tokens   u32 (token_is_u64=0) or u64 (=1) token hashes, 16-byte aligned
 * d_offsets  int64[n_docs+1], non-decreasing CSR offsets, offsets[n_docs] == n_tokens
 * d_init     NULL (empty state, all 0xFFFFFFFF: minhash.py:167-168) or running
 *            signatures to merge (update_batch on a non-empty MinHash, :297);
 *            init_stride = elements between rows (0 = one row broadcast to all docs)
 * d_out      [n_docs, num_perm] u32 (out_is_u64=0) or u64 (=1; the reference's dtype)
 * flags      DSK_KERNEL_*  */
DSK_API int dsk_minhash_bulk(const dsk_perm *perm, const void *d_tokens, int token_is_u64,
                     const int64_t *d_offsets, int64_t n_docs, int64_t n_tokens,
                     const void *d_init, int64_t init_stride, int init_is_u64,
                     void *d_out, int out_is_u64, int flags, void *stream);

/* Same, with a caller-provided device workspace that lets the library cut LONG documents (> 4096 tokens) into pieces
 * of 1024 tokens on the device: the warp that meets such a document stores the row's initial value and appends the
 * pieces to a table in the workspace; a second launch spreads the pieces over all warps and min-merges their partial
 * signatures into the row (atomicMin; MinHash.merge is the combine rule, minhash.py:337-359).  Without a workspace
 * (dsk_minhash_bulk) one warp handles a whole document, whatever its length.  d_workspace: 16-byte aligned,
 * >= dsk_minhash_bulk_workspace_size(n_docs, n_tokens) bytes (0 when no document can be long), contents undefined on
 * entry and on return, owned by the caller, in use until the launch has finished on `stream`.
 * The reference's own GPU benchmark shape is one 50 000-token update_batch (benchmark/sketches/minhash_gpu_benchmark.py:42-48). */
DSK_API size_t dsk_minhash_bulk_workspace_size(int64_t n_docs, int64_t n_tokens);
DSK_API int dsk_minhash_bulk_ws(const dsk_perm *perm, const void *d_tokens, int token_is_u64,
                        const int64_t *d_offsets, int64_t n_docs, int64_t n_tokens,
                        const void *d_init, int64_t init_stride, int init_is_u64,
                        void *d_out, int out_is_u64, int flags, void *d_workspace, size_t workspace_bytes, void *stream);

/* Fused signature build + all-gather (multi-GPU): like dsk_minhash_bulk, but each signature row
 * is stored straight into row (row_offset + i) of the FULL [N_total, num_perm] matrix of every
 * rank: h_peer_out[0..n_peers) are device pointers to those matrices (this rank's own buffer
 * and its peers' buffers mapped over NVLink, e.g. torch symmetric memory / cudaIpc).  The
 * transfer overlaps the integer math document by document; the caller synchronises the ranks
 * afterwards (stream sync + barrier).  Replaces "build, then ncclAllGather". */
DSK_API int dsk_minhash_bulk_gather(const dsk_perm *perm, const void *d_tokens, int token_is_u64,
                                    const int64_t *d_offsets, int64_t n_docs, int64_t n_tokens,
                                    void *const *h_peer_out, int n_peers, int64_t row_offset,
                                    int out_is_u64, int flags, void *stream);

/* Host-buffer variant: same computation, tokens/offsets/out are HOST pointers
 * (pinned memory gives full PCIe overlap; pageable memory is staged).  Documents
 * are cut into slices and H2D copy, kernel and D2H copy are pipelined over
 * internal streams; returns after the last slice landed in h_out.
 * This is the call the reference-facing MinHash.bulk makes. */
DSK_API int dsk_minhash_bulk_host(const dsk_perm *perm, const void *h_tokens, int token_is_u64,
                          const int64_t *h_offsets, int64_t n_docs,
                          const void *h_init, int64_t init_stride, int init_is_u64,
                          void *h_out, int out_is_u64, int flags);

/* Ownership (see INTEGRATION.md "What the library allocates"): every d_ / h_ buffer above is the caller's.  The
 * library itself holds (a) per dsk_perm handle: the permutation table, 16 KB of work counters and 64 events, freed by
 * dsk_perm_destroy; (b) per device, created by the first dsk_minhash_bulk_host call and grown on demand: three
 * streams and three slots of device + pinned staging buffers sized to the largest slice seen (<= 16 Mi tokens,
 * <= 128 Ki documents per slice).  dsk_release_host_pipeline frees (b) for `device` (-1 = every device); the next
 * host-buffer call re-creates it.  Not to be called concurrently with dsk_minhash_bulk_host on the same device. */
DSK_API int dsk_release_host_pipeline(int device);

/* Element-wise min of two signature matrices (MinHash.merge / union,
 * datasketch/minhash.py:359, :453; LeanMinHash.union lean_minhash.py:249). */
DSK_API int dsk_sig_merge_min(const uint32_t *d_x, const uint32_t *d_y, int64_t n_elems, uint32_t *d_out, void *stream);

/* ---- signature codecs (HBM-bound) ---------------------------------------------------
 * LeanMinHash records: `struct` layout "<bo> q i {K}I" = seed int64, K int32, K x uint32
 * (datasketch/lean_minhash.py:174-175 serialize, :201-214 deserialize, :216-232 pickle
 * state).  big_endian = 0 for byteorder '<' '=' '@' (x86-64: 12 + 4K bytes, no padding),
 * 1 for '>' '!'.  d_rec is [n, 12 + 4K] bytes.  Unpack validates every header against
 * (seed, K) and sets *d_status = 1 on a mismatch (d_status must be zeroed by the caller). */
DSK_API int dsk_lean_pack(const void *d_sig, int sig_is_u64, int64_t n, int num_perm, int64_t seed, int big_endian,
                          uint8_t *d_rec, void *stream);
DSK_API int dsk_lean_unpack(const uint8_t *d_rec, int64_t n, int num_perm, int64_t seed, int big_endian, void *d_sig,
                            int sig_is_u64, int *d_status, void *stream);

/* MinHashLSH band keys: for document i and band j, the r hash values
 * sig[i][j*r:(j+1)*r] as big-endian uint64 -- byte-identical to the reference's default
 * `_H` = bytes(hashvalues[start:end].byteswap().data) (datasketch/lsh.py:344, :427, :537-538).
 * d_keys is [n, b, 8*r] bytes. */
DSK_API int dsk_band_keys(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint8_t *d_keys, void *stream);

/* 64-bit fingerprint of each band's r-tuple, [n, b] uint64: the bucket key of the GPU LSH
 * index (equal tuples <=> equal fingerprints up to hash collisions, which the LSH kernels
 * resolve by comparing the tuples themselves). */
DSK_API int dsk_band_fingerprints(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint64_t *d_fp,
                                  void *stream);

/* ---- MinHashLSHBloom ("next" row, SURVEY.md 8f rank 3) -----------------------------------------------
 * dsk_band_sums: the Bloom key of every band, d_keys[i][j] = sum(sig[i][j*r:(j+1)*r]) % (2^61 - 1) as uint64
 * ([n, b]) -- BloomTable.insert / query's `x = sum(hashvalues) % _mersenne_prime`
 * (datasketch/lsh_bloom.py:94-106, :108-118, :20).  HBM-bound codec: 4*num_perm bytes in, 8*b out per document.
 * dsk_bloom_insert / dsk_bloom_query: the same keys go straight into / are tested against b device-resident
 * Bloom tables (MinHashLSHBloom._insert :308-316, query :365-371: a hit in ANY band flags the document).
 * d_bits is [b][words_per_table] uint32, caller-owned and zero-initialised; each key sets / tests n_hashes
 * bits among the table's first n_bits bits (double hashing).  The reference delegates the bit tables to
 * pybloomfilter; these are the library's own (no false negatives, the usual (1 - e^(-kn/m))^k false-positive
 * rate), not pybloomfilter's file format.  d_hit is [n] uint8 (1 = duplicate candidate). */
DSK_API int dsk_band_sums(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint64_t *d_keys, void *stream);
DSK_API int dsk_bloom_insert(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint32_t *d_bits,
                             uint64_t words_per_table, uint64_t n_bits, int n_hashes, void *stream);
DSK_API int dsk_bloom_query(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, const uint32_t *d_bits,
                            uint64_t words_per_table, uint64_t n_bits, int n_hashes, uint8_t *d_hit, void *stream);
/* dsk_bloom_unique: the loop `for each row j in order: if not query(row j): insert(row j)` over a whole batch, on the
 * device.  d_keep[j] = 1 iff the loop inserts row j, and d_bits afterwards hold exactly the bits the loop leaves (the
 * prior bits plus dsk_bloom_insert of the kept rows), Bloom false positives included.  Stream-ordered, no host
 * synchronisation.  d_sig 4-byte aligned; d_ws 16-byte aligned and at least dsk_bloom_unique_workspace_size() bytes:
 * with E = n * b * n_hashes probe entries, 24*E (key table at load factor 1/2) + 8*E (entry slots and links) + 12*n
 * bytes, each of its 8 parts rounded up to 256.  The workspace size is 0 for n <= 0, for invalid (num_perm, b, r,
 * n_hashes) and for E > 2^30, which dsk_bloom_unique rejects (split the batch: consecutive calls give the same result as
 * one call over their concatenation).  n_bits must satisfy b * n_bits < 2^64. */
DSK_API size_t dsk_bloom_unique_workspace_size(int64_t n, int num_perm, int b, int r, int n_hashes);
DSK_API int dsk_bloom_unique(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint32_t *d_bits,
                             uint64_t words_per_table, uint64_t n_bits, int n_hashes, void *d_ws, size_t ws_bytes,
                             uint8_t *d_keep, void *stream);

/* ---- Weighted MinHash (Ioffe ICWS) ------------------------------------------------------
 * Handle = device copy of the generator parameters rs, ln_cs, betas, each [sample_size, dim]
 * float32, drawn on the HOST by numpy exactly as WeightedMinHashGenerator.__init__ does
 * (datasketch/weighted_minhash.py:118-121).  dsk_wmh_minhash replaces the per-sample loop
 * of WeightedMinHashGenerator.minhash (:147-158) for a batch of n vectors:
 *   d_v      [n, dim] float32 weights (zeros are skipped, :148-152)
 *   d_out    [n, sample_size, 2] int64: (k, int(t_k)) per sample (:158); a non-finite t_k (a +inf weight, or a NaN
 *            winner in MINHASH_MANY) is stored as INT64_MIN, numpy's float -> int64 cast on x86-64
 *   d_status [n] int32: 0; 1 where the row has no candidate column: all zeros (reference: ValueError, :149-150), or
 *            in minhash mode all zeros, negative or NaN (ValueError from np.nanargmin); 2 where t_k is not finite in
 *            every sample (reference: OverflowError from int(t), :158)
 *   flags    DSK_WMH_MINHASH (0): np.nanargmin, so negative and NaN weights are skipped like zeros;
 *            or DSK_WMH_MINHASH_MANY: the float32 operation order of the reference's experimental minhash_many
 *            (:221-224) and np.argmin over the non-zero columns, where the first negative or NaN weight wins (an
 *            all-zero row is None there, :241-245)
 *            | DSK_WMH_INPUT_LOG: d_v holds ln(weight) already (float32, -inf where the weight is zero) -- the host
 *            layer passes numpy's own float32 log (:152), which makes every step bit-identical to the reference;
 *            without it the kernel takes log() in double rounded to float32 itself (the correctly rounded float32
 *            log except within a few double ulps of a rounding midpoint; numpy's differs from it by up to 3 ulp) */
#define DSK_WMH_MINHASH 0
#define DSK_WMH_MINHASH_MANY 1
#define DSK_WMH_INPUT_LOG 2
typedef struct dsk_wmh dsk_wmh;
DSK_API int dsk_wmh_create(const float *h_rs, const float *h_ln_cs, const float *h_betas, int sample_size, int dim,
                           int device, dsk_wmh **out);
DSK_API void dsk_wmh_destroy(dsk_wmh *g);
DSK_API int dsk_wmh_minhash(const dsk_wmh *g, const float *d_v, int64_t n, int64_t *d_out, int32_t *d_status,
                            int flags, void *stream);
/* dsk_wmh_minhash_csr: the same sampling for n SPARSE rows in CSR form, in time linear in their stored entries (the
 * sparse path of the reference's minhash_many, :191-239, without densifying).  Row i holds the entries
 * [d_indptr[i], d_indptr[i + 1]) of d_indices (column) and d_vals (weight, or ln(weight) with DSK_WMH_INPUT_LOG).
 *   d_indptr  [n + 1] int64: must start at 0 and be non-decreasing (not checked here: the kernel reads the entries it
 *             names; the host layer checks it before the call)
 *   d_indices [nnz] int32: strictly increasing within each row, each in [0, dim); a row that breaks this gets status 3
 *             and (0, 0) in every sample, and is not evaluated further
 *   d_out, d_status, flags: as dsk_wmh_minhash.  Each row's result equals dsk_wmh_minhash on the densified row bit for
 *             bit: a left-out column is a zero weight, which never wins, and explicit zeros may be stored.
 * n == 0 is a no-op (the buffers may then be NULL); for n > 0 every pointer must be non-NULL. */
DSK_API int dsk_wmh_minhash_csr(const dsk_wmh *g, const int64_t *d_indptr, const int32_t *d_indices, const float *d_vals,
                                int64_t n, int64_t *d_out, int32_t *d_status, int flags, void *stream);

/* ---- device-resident MinHashLSH index ------------------------------------------------------
 * Replaces the bucket step of MinHashLSH._insert / query over dict storage
 * (datasketch/lsh.py:344-347, :426-429; storage.py:209-259) for whole batches.  Documents are
 * numbered 0..n_docs-1 in insertion order (the host layer maps numbers to user keys).  Buckets
 * are exact: two documents meet iff a band's r-tuple is equal, as with the reference's byte keys.
 *   dsk_lsh_insert       append n signatures ([n, num_perm] u32) to the index
 *   dsk_lsh_insert_tokens  the same from TOKENS: builds the n documents' signatures (dsk_minhash_bulk's kernel) straight into
 *                        the index's own signature storage and inserts each document in the same launch -- the warp that
 *                        finishes a row does its b bucket updates, whose DRAM latency hides behind the other warps'
 *                        integer work; the signature matrix is never read back.  (MinHash.bulk + MinHashLSH.insert per
 *                        document, minhash.py:464-489 + lsh.py:326-347.)  Fused for u32 tokens, a handle with
 *                        n_unsafe == 0 and num_perm <= 256; any other input runs the two kernels one after the other.
 *   dsk_lsh_query_count  d_counts[q] = number of distinct candidates of query q
 *   dsk_exclusive_scan   d_out[0..n] = exclusive prefix sums of d_in[0..n-1] (d_out[n] = total);
 *                        d_scratch holds at least n/1024 + 2 int64
 *   dsk_lsh_query_fill   writes each query's candidates (document numbers, unordered like the
 *                        reference's list(set), lsh.py:432) at d_idx[d_ptr[q] .. d_ptr[q+1])
 * Self-join of the n_docs documents inserted so far.  i and d < i are a candidate pair iff d is a candidate of
 * query(row i), and eq(i, d) = number of the num_perm positions where the two rows agree (MinHash.jaccard * num_perm,
 * minhash.py:324).  min_count in [0, num_perm] keeps the pairs with eq >= min_count (0 keeps all).
 *   dsk_lsh_pairs_count  d_counts[i] = number of kept partners d < i of document i
 *   dsk_lsh_pairs_fill   after dsk_exclusive_scan of the counts: writes i's partners at d_idx[d_ptr[i] .. d_ptr[i+1])
 *                        (unordered) and their eq at the same positions of d_eq
 *   dsk_lsh_clusters     d_labels[i] = smallest document number of i's connected component of the kept pairs' graph
 *                        (deterministic; d_labels is the union-find's parent array, no other workspace).  min_count = 0
 *                        links each document to the first equal member of each of its buckets: linear in the index.
 *                        min_count > 0 walks every pair: quadratic in the size of each bucket.
 * Removal (MinHashLSH.remove, lsh.py:509-528).  A removed document keeps its number until dsk_lsh_compact, and n_docs
 * (dsk_lsh_size) still counts it.  query never returns it, the self-join pairs nothing with it (its own count is 0) and
 * dsk_lsh_clusters labels it -1; pairs among the remaining documents are exactly those before the removal.  An index that
 * never removed anything, or whose removals were compacted, runs the same kernels as before removal existed.
 *   dsk_lsh_remove       marks the n documents d_docs[0..n) removed (asynchronous, ordered on the stream; the first call
 *                        allocates a bitmap of capacity_docs bits).  d_status[0] += ids outside [0, n_docs), which are
 *                        ignored; d_status[1] += ids already removed, a repeat within d_docs included.  Idempotent.
 *   dsk_lsh_alive        d_out[j] = 1 iff d_docs[j] is in [0, n_docs) and not removed, else 0
 *   dsk_lsh_compact      renumbers the remaining documents 0..m-1 in their old order and rebuilds the bucket tables from
 *                        them: d_remap[old] = new number, or -1 for a removed document (n_docs entries).  The rows move
 *                        inside the index's own storage, so the freed capacity can be inserted again.  Afterwards the index
 *                        behaves as a fresh one into which the remaining rows were inserted in order.  The call
 *                        SYNCHRONISES the stream once, to read m, and then sets n_docs = m; with nothing removed since
 *                        the last compaction it writes the identity remap and returns without synchronising.
 *   dsk_lsh_compact_workspace_size  bytes of d_ws (16-byte aligned) for the index's current n_docs: the removal bitmap's
 *                        per-word prefix counts, the new -> old index (int32 per document) and a fixed staging area of
 *                        at most 64 MB for the rows.  It does not grow as n_docs * num_perm. */
typedef struct dsk_lsh dsk_lsh;
DSK_API int dsk_lsh_create(int num_perm, int b, int r, int64_t capacity_docs, int device, dsk_lsh **out);
/* An index of WEIGHTED MinHash signatures (MinHashLSH over WeightedMinHash, lsh.py:344, weighted_minhash.py:55-60).  A row
 * is [2 * sample_size] u32: sample j's (k_j, t_j) pair is word 2j = k_j as uint32 and word 2j + 1 = t_j as int32 (two's
 * complement).  On 0 <= k < 2^32, -2^31 <= t < 2^31 this packing is injective, so two bands of r samples have equal
 * reference keys (the byteswapped int64 pairs) iff their 2r words are equal, and band j of the reference is band j of a
 * (b, 2r) banding over 2 * sample_size words.  b and r count samples (b * r <= sample_size).  Every entry below takes such
 * rows in place of [n, num_perm] ones (dsk_lsh_insert, dsk_lsh_query_*, dsk_lsh_unique_*; the d_sig of dsk_lsh_unique_*
 * must be 8-byte aligned), min_count is in [0, sample_size] and every eq counts SAMPLES whose two words both agree, so
 * eq / sample_size is WeightedMinHash.jaccard.  dsk_lsh_insert_tokens returns DSK_ERR_INVALID for such an index. */
DSK_API int dsk_lsh_create_weighted(int sample_size, int b, int r, int64_t capacity_docs, int device, dsk_lsh **out);
DSK_API void dsk_lsh_destroy(dsk_lsh *ix);
DSK_API int dsk_lsh_size(const dsk_lsh *ix, int64_t *n_docs, int64_t *capacity_docs);
DSK_API int dsk_lsh_insert(dsk_lsh *ix, const uint32_t *d_sig, int64_t n, void *stream);
DSK_API int dsk_lsh_insert_tokens(dsk_lsh *ix, const dsk_perm *perm, const void *d_tokens, int token_is_u64,
                                  const int64_t *d_offsets, int64_t n_docs, int64_t n_tokens, void *stream);
DSK_API int dsk_lsh_query_count(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_query_fill(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, const int64_t *d_ptr,
                               int32_t *d_idx, void *stream);
DSK_API int dsk_exclusive_scan(const int64_t *d_in, int64_t n, int64_t *d_out, int64_t *d_scratch, void *stream);
DSK_API int dsk_lsh_pairs_count(const dsk_lsh *ix, int min_count, int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_pairs_fill(const dsk_lsh *ix, int min_count, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                               void *stream);
DSK_API int dsk_lsh_clusters(const dsk_lsh *ix, int min_count, int32_t *d_labels, void *stream);
/* Query rows that are NOT in the index, verified on the device (MinHashLSH.query + MinHash.jaccard per candidate,
 * lsh.py:370-432, minhash.py:299-324): the self-join's walk with the query row staged in place of document i and every
 * document d < n_docs eligible.  d_qsig is [nq, num_perm] u32; min_count in [0, num_perm] keeps the candidates with
 * eq >= min_count, where eq = number of positions where the query row and the document's row agree.  Removed documents
 * (since the last dsk_lsh_compact) are never returned.  nq == 0 with null buffers is a valid no-op.  A query that hits a
 * bucket of s members reads up to s rows of num_perm words: its time is linear in the size of the buckets it hits.
 *   dsk_lsh_query_jaccard_count  d_counts[q] = number of kept candidates of query q
 *   dsk_lsh_query_jaccard_fill   after dsk_exclusive_scan of the counts: writes q's kept candidates (each once, unordered)
 *                                at d_idx[d_ptr[q] .. d_ptr[q+1]) and their eq at the same positions of d_eq.  Without a
 *                                filter the candidates are exactly dsk_lsh_query_fill's.
 *   dsk_lsh_query_best           d_idx[q] / d_eq[q] = q's kept candidate with the largest eq, the smallest document number
 *                                among equal ones (deterministic); -1 / -1 when q keeps none.  One launch: no count, scan
 *                                or fill, no synchronisation. */
DSK_API int dsk_lsh_query_jaccard_count(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count,
                                        int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_query_jaccard_fill(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count,
                                       const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq, void *stream);
DSK_API int dsk_lsh_query_best(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int32_t *d_idx,
                               int32_t *d_eq, void *stream);
/* The k most similar kept candidates of each row, ranked on the device (the candidates of dsk_lsh_query_jaccard_fill, sorted
 * by eq descending, then document number ascending, and cut at k).  k in [1, 32]; min_count as above.  Row q's list is at
 * d_idx[q * k .. q * k + k) with its eq at the same positions of d_eq, best first; the slots behind the last kept candidate
 * hold -1 / -1.  Removed documents (since the last dsk_lsh_compact) are never listed.  One launch: no count, scan or fill,
 * no workspace, no synchronisation.  The walk and the verification are dsk_lsh_query_jaccard_count's; only the output is
 * bounded (k entries per row).
 *   dsk_lsh_query_topk   d_qsig [nq, num_perm] u32 query rows, d_idx / d_eq [nq, k].  k = 1 gives dsk_lsh_query_best.
 *                        nq == 0 with null buffers is a valid no-op.
 *   dsk_lsh_neighbors    every document i's own row against every other document d != i (d < i and d > i): i's k nearest
 *                        neighbours, d_idx / d_eq [n_docs, k].  A removed document's row is all -1.  Each pair is verified
 *                        from both ends, about twice dsk_lsh_pairs_count's row comparisons.  An empty index with null
 *                        buffers is a valid no-op. */
DSK_API int dsk_lsh_query_topk(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int k, int32_t *d_idx,
                               int32_t *d_eq, void *stream);
DSK_API int dsk_lsh_neighbors(const dsk_lsh *ix, int min_count, int k, int32_t *d_idx, int32_t *d_eq, void *stream);
/* Streaming de-duplication of a batch (the loop `for m in batch: if not [d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]:
 * lsh.insert(key, m)`, lsh.py:326-347 / :370-432, minhash.py:299-324), on the device.  Row j of d_sig ([n, num_perm] u32)
 * is KEPT iff no remaining (not removed) document of the index and no row j' < j of the batch that was kept is a candidate
 * of row j with eq >= min_count (min_count in [0, num_perm]; 0: any candidate drops the row).  The kept rows are inserted in
 * batch order as documents n_docs, n_docs + 1, ...; afterwards the index equals one into which the loop inserted them.
 *   dsk_lsh_unique_workspace_size  bytes of d_ws (16-byte aligned) for n rows: the batch's own bucket table, cap_slots =
 *                        the smallest power of two >= 2n (at least 2), i.e. 16 * b * cap_slots + 4 * b * n bytes, about
 *                        32 * b * n + 4 * b * n; plus about 40 * n bytes for stage A's idx / eq, the statuses, the kept flags and
 *                        their scan, two row lists and new -> old; each part rounded up to 256 bytes.  0 for n <= 0.
 *   dsk_lsh_unique_count builds the batch table over d_sig, walks every row against the index (the best kept candidate
 *                        there, as dsk_lsh_query_best) and writes d_counts[j] = the number of rows d < j of the batch that
 *                        are candidates of row j with eq >= min_count.  Asynchronous, no synchronisation.
 *   dsk_lsh_unique_commit after dsk_exclusive_scan of the counts into d_ptr (n + 1 entries): writes the batch pairs into
 *                        d_pidx / d_peq (d_ptr[n] entries each), resolves the loop's decisions, then writes d_kept[j]
 *                        (1 / 0) and, for a dropped row, d_match[j] / d_eq[j] = the candidate of the loop's query with the
 *                        largest eq, the smallest document number among equal ones (numbers after the call: indexed
 *                        documents win ties against batch rows); -1 / -1 for a kept row.  It SYNCHRONISES the stream once,
 *                        to read the number m of kept rows; if n_docs + m > capacity_docs it returns DSK_ERR_INVALID with
 *                        the index unchanged (the outputs are written), else it inserts the kept rows and sets
 *                        *h_inserted = m (host memory).
 * The commit must follow the count with the same d_sig, n, min_count and d_ws (the workspace carries the batch table and
 * stage A's results between them) and with no change of the index in between; anything else is DSK_ERR_INVALID.  Both
 * check the handle, n >= 0, min_count, the workspace and the buffers; n == 0 with null buffers is a valid no-op.  Cost: the
 * batch walk is quadratic in the size of each within-batch bucket (as dsk_lsh_pairs_* with min_count > 0); the resolution
 * takes about as many rounds as the longest chain of rows whose decisions wait for each other (a drift chain of L rows:
 * ~L rounds), run by one CTA after three grid-wide sweeps, without host synchronisation. */
DSK_API size_t dsk_lsh_unique_workspace_size(const dsk_lsh *ix, int64_t n);
DSK_API int dsk_lsh_unique_count(const dsk_lsh *ix, const uint32_t *d_sig, int64_t n, int min_count, void *d_ws,
                                 size_t ws_bytes, int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_unique_commit(dsk_lsh *ix, const uint32_t *d_sig, int64_t n, int min_count, void *d_ws, size_t ws_bytes,
                                  const int64_t *d_ptr, int32_t *d_pidx, int32_t *d_peq, uint8_t *d_kept, int32_t *d_match,
                                  int32_t *d_eq, int64_t *h_inserted, void *stream);
/* ---- device-resident MinHashLSHEnsemble (containment search) -------------------------------------------------------
 * Replaces MinHashLSHEnsemble.index / query over dict storage (datasketch/lshensemble.py:189-249): num_part x |rs|
 * MinHashLSH indexes filled per set and walked per query in Python.  The host computes what is control logic there and
 * passes it in: the (b, r) table params (lshensemble.py:155-166, 10 rows), the size partitions and, per query and
 * partition, the row of that table the query uses.
 *   dsk_lsh_ensemble_create  h_b / h_r: the n_params (<= 16) rows of the (b, r) table, b*r <= num_perm.  For each distinct
 *                        r the index keeps one set of b_r = num_perm / r band tables, as the reference's
 *                        MinHashLSH(params=(num_perm / r, r)).  Allocates no device memory.
 *   dsk_lsh_ensemble_index  indexes the n sets of d_sig ([n, num_perm] u32), once (a second call is DSK_ERR_INVALID).
 *                        d_order[t] (a permutation of 0..n-1) is the row of d_sig that becomes set number t: the rows in
 *                        stable size order, as the reference's entries.sort(key=size).  h_part_start[0..num_part] (host
 *                        memory, rising from 0 to n): partition p holds set numbers [h_part_start[p], h_part_start[p+1]).
 *                        A set matches another in band j of table set r iff both are in the same partition and their
 *                        r-tuples in band j are equal (the bucket indexes[p][r].hashtables[j][H] of the reference).  It
 *                        allocates, synchronously, dsk_lsh_ensemble_index_bytes(n) bytes of device memory:
 *                          4 * num_perm * n              the rows, once, in size order
 *                        + 4 * n + 8 * (num_part + 1)    the map set number -> row of d_sig, the partition bounds
 *                        + sum over distinct r of b_r * (16 * cap_slots + 4 * n),  cap_slots = the power of two >= 2n
 *                        (e.g. threshold 0.5, num_perm 128, m 8: rs = {1, 2, 3, 5, 8}, sum b_r = 275, about 11 GB at 1M
 *                        sets).  If it cannot, it returns DSK_ERR_NOMEM and the handle stays empty and usable.
 *   dsk_lsh_ensemble_query_count  d_sel[q * num_part + p] = the row of the (b, r) table query q uses in partition p
 *                        (lshensemble.py:162-166: searchsorted(xqs, upper_p / size_q) clamped to the last row), or -1 to
 *                        skip the partition (upper bound None); any value outside [0, n_params) skips it too.  Writes
 *                        d_counts[q * num_part + p] = the number of candidates of q in p: the sets of p that share the
 *                        query's r-tuple in one of the first b bands of the (num_perm / r, r) banding (MinHashLSH._query_b).
 *   dsk_exclusive_scan   of the nq * num_part counts into d_ptr (nq * num_part + 1 entries)
 *   dsk_lsh_ensemble_query_fill  writes the candidates of item q * num_part + p, each once, unordered, as rows of the
 *                        index call's d_sig, at d_idx[d_ptr[item] .. d_ptr[item + 1]); q's whole result is
 *                        d_idx[d_ptr[q * num_part] .. d_ptr[(q + 1) * num_part]).  d_eq (may be NULL): at the same
 *                        positions, the number of the num_perm positions where the query row and the set's row agree.
 * Queries check the handle, nq >= 0 and, for nq > 0, every buffer; nq == 0 with null buffers is a valid no-op, and an
 * index that was never built has no candidates.  Cost: one warp per (query, partition) probes b tables of one set and
 * walks the chains it hits, reading the r-tuple of each member (and, with d_eq, both rows of each candidate).
 * Containment estimates of the candidates.  For query q of size s_q and candidate x (a row of the index call) of size s_x,
 * with j = eq / num_perm (MinHash.jaccard): c = j * (s_q + s_x) / (s_q * (1 + j)), the inverse of the map from containment t
 * to the Jaccard value t / (1 + s_x/s_q - t) that the (b, r) table was chosen for, so c estimates |Q & X| / |Q|.  It is
 * computed in float64 bit for bit as that Python expression over ints and floats (each operation rounded on its own, s_q + s_x
 * summed exactly) and not clamped: c exceeds 1 when s_x > s_q and j is near 1.  A candidate is kept iff c >= min_containment
 * (in [0, 1]; 0 keeps every candidate, since c >= 0).  d_qsizes: int64[nq], each in [1, 2^62); d_set_sizes: int64[n], the
 * index call's sizes in its row order (the caller keeps them on the device; the index holds its rows in size order only).
 *   dsk_lsh_ensemble_containment_count  d_counts[q * num_part + p] = the number of kept candidates of q in p (the candidates
 *                        of dsk_lsh_ensemble_query_count, each with its eq counted when min_containment > 0).
 *   dsk_lsh_ensemble_containment_fill  after dsk_exclusive_scan of those counts into d_ptr: the kept candidates of each item,
 *                        each once, unordered, at d_idx[d_ptr[item] ..), with d_eq and d_containment (float64) at the same
 *                        positions.  With min_containment = 0 the (idx, eq) pairs are those of dsk_lsh_ensemble_query_fill.
 *   dsk_lsh_ensemble_containment_topk  for each query, its k (1..32) kept candidates of largest c, ties to the smaller row:
 *                        d_idx / d_eq / d_containment [q * k .. q * k + k), padded with -1 / -1 / -1.0.  One launch, no
 *                        scan: one warp per query walks its partitions in turn and keeps a warp-held list.
 *   dsk_lsh_ensemble_self_containment_count / _fill  the self-join: the same for each indexed set i as a query (its own row
 *                        and size d_set_sizes[i]), set i itself left out by identity (an equal row of equal size is still
 *                        listed).  d_sel is [n, num_part] in the index call's row order (built from the indexed sizes), the
 *                        items are i * num_part + p in that order, and nothing is read but the index's own rows.  An index
 *                        never built is a no-op.
 * Each returns DSK_ERR_INVALID with a message for a null handle, nq < 0, a null buffer when there is work (nq > 0, or n > 0
 * for the self-join), k outside [1, 32], and min_containment NaN or outside [0, 1]; nq == 0 with null buffers is a no-op.
 * Cost: the walk of the query functions, plus one K-word row comparison per candidate (the count pass skips it when
 * min_containment is 0) and one int64 size read. */
typedef struct dsk_lsh_ensemble dsk_lsh_ensemble;
DSK_API int dsk_lsh_ensemble_create(int num_perm, int num_part, const int32_t *h_b, const int32_t *h_r, int n_params,
                                    int device, dsk_lsh_ensemble **out);
DSK_API void dsk_lsh_ensemble_destroy(dsk_lsh_ensemble *e);
DSK_API int dsk_lsh_ensemble_size(const dsk_lsh_ensemble *e, int64_t *n_sets);
DSK_API size_t dsk_lsh_ensemble_index_bytes(const dsk_lsh_ensemble *e, int64_t n_sets);
DSK_API int dsk_lsh_ensemble_index(dsk_lsh_ensemble *e, const uint32_t *d_sig, int64_t n, const int32_t *d_order,
                                   const int64_t *h_part_start, void *stream);
DSK_API int dsk_lsh_ensemble_query_count(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int32_t *d_sel,
                                         int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_ensemble_query_fill(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int32_t *d_sel,
                                        const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq, void *stream);
DSK_API int dsk_lsh_ensemble_containment_count(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq,
                                               const int64_t *d_qsizes, const int32_t *d_sel, const int64_t *d_set_sizes,
                                               double min_containment, int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_ensemble_containment_fill(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq,
                                              const int64_t *d_qsizes, const int32_t *d_sel, const int64_t *d_set_sizes,
                                              double min_containment, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                                              double *d_containment, void *stream);
DSK_API int dsk_lsh_ensemble_containment_topk(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq,
                                              const int64_t *d_qsizes, const int32_t *d_sel, const int64_t *d_set_sizes,
                                              double min_containment, int k, int32_t *d_idx, int32_t *d_eq,
                                              double *d_containment, void *stream);
DSK_API int dsk_lsh_ensemble_self_containment_count(const dsk_lsh_ensemble *e, const int32_t *d_sel, const int64_t *d_set_sizes,
                                                    double min_containment, int64_t *d_counts, void *stream);
DSK_API int dsk_lsh_ensemble_self_containment_fill(const dsk_lsh_ensemble *e, const int32_t *d_sel, const int64_t *d_set_sizes,
                                                   double min_containment, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                                                   double *d_containment, void *stream);
/* The size partitions of MinHashLSHEnsemble.index (lshensemble_partition.py:54-196, optimal_partitions), on the device.
 * h_sizes / h_counts (host memory, n_sizes = D entries): the distinct set sizes, strictly ascending, and their counts, every
 * value in [1, 2^62).  Writes h_upper_idx[k] (host memory, min(num_part, D) entries) = the index into h_sizes of the upper
 * bound of partition k; partition k covers sizes (h_upper_idx[k-1], h_upper_idx[k]] (from index 0 for k = 0), the last ends
 * at D - 1.  These are the reference's bounds bit for bit: cost[l, u] = sum over i in [l, u] of (sizes[u] - sizes[i]) /
 * sizes[u] * counts[i] with each operation rounded on its own and numpy's float64 pairwise summation, the reference's
 * dynamic programme (its back-tracking reads the p-interval table where the recurrence used p - 1, reproduced), and every
 * argmin takes the first index among equal values.
 *   dsk_ensemble_partition_workspace_size  bytes of d_workspace (16-byte aligned), each part rounded up to 256 bytes:
 *                        16 * D (sizes, counts); for D > 28672 also 8 * D * min(D, 512) (terms of the cost columns, which
 *                        fit shared memory below); for 2 <= num_part < D also 4 * D * (D + 1) (the cost triangle, 50 MB at
 *                        D = 3550, 1.6 GB at D = 20000) + 8 * D * (num_part - 1) (the tables) + 8 * num_part.  0 for
 *                        n_sizes < 1 or num_part < 1; SIZE_MAX if the sum does not fit in size_t.
 *   dsk_ensemble_partition  num_part < 2 (one partition) and num_part >= D (one per size) need no table: the bounds are
 *                        written on the host, with no device work and no workspace, unless d_cost is given.  Otherwise it
 *                        copies sizes and counts to the device, fills the triangle, runs num_part - 2 launches of the
 *                        programme and one of the back-tracking, copies the num_part indices back and synchronises the
 *                        stream once, at the end.  d_cost (may be NULL; device memory, D(D+1)/2 doubles): the triangle is
 *                        written there instead of the workspace, entry (l, u) at u(u+1)/2 + l, in every case.
 *                        DSK_ERR_INVALID (with a message) for n_sizes < 1, num_part < 1, null host buffers, sizes not
 *                        strictly ascending or outside [1, 2^62), counts outside [1, 2^62), and a workspace that is too
 *                        small or not 16-byte aligned.
 * Cost: D^3/6 float64 additions and D^2/2 divisions for the triangle (one CTA per column, one thread per entry, the column's
 * terms shared), then num_part reads of it. */
DSK_API size_t dsk_ensemble_partition_workspace_size(int64_t n_sizes, int num_part);
DSK_API int dsk_ensemble_partition(const int64_t *h_sizes, const int64_t *h_counts, int64_t n_sizes, int num_part,
                                   void *d_workspace, size_t workspace_bytes, int device, int64_t *h_upper_idx,
                                   double *d_cost, void *stream);
DSK_API int dsk_lsh_remove(dsk_lsh *ix, const int32_t *d_docs, int64_t n, int64_t *d_status, void *stream);
DSK_API int dsk_lsh_alive(const dsk_lsh *ix, const int32_t *d_docs, int64_t n, uint8_t *d_out, void *stream);
DSK_API size_t dsk_lsh_compact_workspace_size(const dsk_lsh *ix);
DSK_API int dsk_lsh_compact(dsk_lsh *ix, int32_t *d_remap, void *d_ws, size_t ws_bytes, void *stream);

/* ---- Jaccard estimate -----------------------------------------------------------------------
 * d_count[p] = number of positions where rows d_i[p] and d_j[p] of the [n_rows, num_perm] u32
 * signature matrix are equal; jaccard = count / num_perm (MinHash.jaccard,
 * datasketch/minhash.py:324; seeds / lengths are validated by the host layer as :314-323).
 * An out-of-range pair index yields -1. */
DSK_API int dsk_jaccard_pairs(const uint32_t *d_sig, int64_t n_rows, int num_perm, const int64_t *d_i,
                              const int64_t *d_j, int64_t m, int32_t *d_count, void *stream);

/* All-pairs top-k: for each of nq query rows, the `topk` (<= 32) rows of the [n, num_perm]
 * database with the most equal positions, best first; ties -> lower database index.  If
 * self_base >= 0, query i is database row self_base + i and is excluded from its own list.
 * d_cnt [nq, topk] int32 counts (jaccard = cnt / num_perm), d_idx [nq, topk] int64 (-1 pads). */
DSK_API int dsk_jaccard_topk(const uint32_t *d_q, int64_t nq, const uint32_t *d_db, int64_t n, int num_perm, int topk,
                             int64_t self_base, int32_t *d_cnt, int64_t *d_idx, void *stream);
/* Same result, ~3x fewer ALU ops: with a caller-provided workspace (16-byte aligned, >= dsk_jaccard_topk_workspace_size()
 * bytes -- 0 means the prefilter does not apply (num_perm < 32 or > 480, where a tile pair's planes exceed one block's
 * shared memory, or n < 512) and the call behaves like dsk_jaccard_topk) both matrices are first reduced
 * to bit-sliced 16-bit fingerprints; a pair reaches the exact count only if the fingerprint agreement -- an upper bound of
 * the number of equal positions -- could still enter the query's list.  Lists are identical to dsk_jaccard_topk's. */
DSK_API size_t dsk_jaccard_topk_workspace_size(int64_t nq, int64_t n, int num_perm);
DSK_API int dsk_jaccard_topk_ws(const uint32_t *d_q, int64_t nq, const uint32_t *d_db, int64_t n, int num_perm, int topk,
                                int64_t self_base, int32_t *d_cnt, int64_t *d_idx, void *d_workspace,
                                size_t workspace_bytes, void *stream);

/* ---- LSH Forest query ("next" row, SURVEY.md 8f) ----------------------------------------------
 * d_order is [l, n] int32: for tree t, the document numbers sorted by (sig[doc][t*k:(t+1)*k]
 * lexicographically, document number) -- the flattening of the reference's sorted key list +
 * insertion-ordered buckets (datasketch/lshforest.py:68-72).  For each query the kernel walks
 * prefix lengths r = k..1 and trees 0..l-1 exactly like MinHashLSHForest.query (:74-128) and writes
 * the first `topk` (<= 1024) distinct document numbers it meets (d_out [nq, topk], -1 pads). */
DSK_API int dsk_forest_query(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int l, int k,
                             const uint32_t *d_qsig, int64_t nq, int topk, int32_t *d_out, void *stream);

/* Weighted MinHash rows (MinHashLSHForest over WeightedMinHash): d_sig / d_qsig are [n, 2 * sample_size] u32, sample j
 * packed as word 2j = k_j (uint32) and word 2j + 1 = t_j (int32, two's complement), 8-byte aligned; l, k and
 * sample_size count samples.  Compared as unsigned words, such rows sort like the reference's big-endian int64 (k, t)
 * keys, so d_order is built exactly as above over the tree's 2k words, and the walk compares 2r words for a prefix of
 * r samples.  Otherwise as dsk_forest_query. */
DSK_API int dsk_forest_query_weighted(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int sample_size, int l,
                                      int k, const uint32_t *d_qsig, int64_t nq, int topk, int32_t *d_out, void *stream);
/* Ranked forest queries.  weighted = 0: rows of num_perm words; weighted = 1: rows as dsk_forest_query_weighted's, with
 * num_perm the sample size.  For each query the walk collects the first `candidates` (topk <= candidates <= 1024)
 * distinct documents dsk_forest_query(..., candidates) would return; then eq[d] = the number of positions (samples,
 * whole (k, t) pairs) among all num_perm where the rows agree -- eq / num_perm is MinHash.jaccard / WeightedMinHash.jaccard
 * -- and the collected documents with eq >= min_count (0 <= min_count <= num_perm) are ranked by larger eq, then smaller
 * number.  d_idx / d_eq [nq, topk] (1 <= topk <= 32) hold the first topk of them, -1 / -1 behind.  The filter never
 * changes which documents are collected.  One launch, no workspace. */
DSK_API int dsk_forest_query_topk(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int weighted,
                                  int l, int k, const uint32_t *d_qsig, int64_t nq, int candidates, int min_count, int topk,
                                  int32_t *d_idx, int32_t *d_eq, void *stream);
/* The same ranking for every indexed row i ([n, topk] outputs): the walk of row i collects the first `candidates`
 * distinct documents other than i (by number: an exact copy of i is collected; i never counts against candidates). */
DSK_API int dsk_forest_neighbors(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int weighted,
                                 int l, int k, int candidates, int min_count, int topk, int32_t *d_idx, int32_t *d_eq,
                                 void *stream);

/* ---- b-bit MinHash blocks ("next" row, SURVEY.md 8f) -----------------------------------------
 * bBitMinHash keeps the b lowest bits of each value (datasketch/b_bit_minhash.py:38) and packs
 * them into 64-bit blocks, value j of a block at bit (n-1-j)*slot with slot = 1,2,4,8,16,32 >= b
 * and n = 64/slot (:78-92).  d_blocks is [n, ceil(num_perm / n)] uint64 (the payload after the
 * 21-byte '<qBdi' header of the pickle state). */
DSK_API int dsk_bbit_pack(const uint32_t *d_sig, int64_t n, int num_perm, int b, uint64_t *d_blocks, void *stream);
DSK_API int dsk_bbit_unpack(const uint64_t *d_blocks, int64_t n, int num_perm, int b, uint32_t *d_sig, void *stream);

/* ---- default token hash on device ("next" row, SURVEY.md 8f) --------------------------------
 * d_out[t] = sha1_hash32 (out_is_u64 = 0) or sha1_hash64 (= 1) of the byte string
 * d_bytes[d_byte_offsets[t] : d_byte_offsets[t+1]] -- datasketch/hashfunc.py:5-28, i.e. the
 * first 4 / 8 bytes of SHA-1 read little-endian.  Lets MinHash.bulk with the default hashfunc
 * skip the per-token Python hashlib loop (minhash.py:263). */
DSK_API int dsk_sha1_tokens(const uint8_t *d_bytes, const int64_t *d_byte_offsets, int64_t n_tokens, void *d_out,
                            int out_is_u64, void *stream);

/* ---- fast non-cryptographic token hashes on device ("next" row, SURVEY.md 8f rank 1) -------------
 * The hash functions the reference documents as `hashfunc` alternatives (docs/minhash.rst:79-112):
 *   DSK_HASH_XXH32       XXH32(data, seed)             == xxhash.xxh32_intdigest(data, seed)
 *   DSK_HASH_MURMUR3_32  MurmurHash3_x86_32(data, seed) == mmh3.hash(data, seed, signed=False)
 * d_out[t] = 32-bit hash of d_bytes[d_byte_offsets[t] : d_byte_offsets[t+1]]; replaces the per-token
 * Python call of minhash.py:263 when the user's hashfunc is one of these. */
#define DSK_HASH_XXH32 1
#define DSK_HASH_MURMUR3_32 2
DSK_API int dsk_hash_tokens(const uint8_t *d_bytes, const int64_t *d_byte_offsets, int64_t n_tokens, int kind,
                            uint32_t seed, uint32_t *d_out, void *stream);

/* ---- raw UTF-8 text to word / character n-gram tokens (DESIGN.md §4m) -------------------------------------------------
 * Replaces the user's shingling loop in front of MinHash.bulk; the reference has none and leaves it to the user.  Document
 * i is d_text[d_doc_offsets[i] : d_doc_offsets[i+1]], read as UTF-8 on its own.  Its units are its words (unit
 * DSK_SHINGLE_WORD: str.split() with no argument, i.e. maximal runs of code points outside Python's 29 whitespace code
 * points) or its code points (DSK_SHINGLE_CHAR).  With m units it has max(m - n + 1, min(m, 1)) shingles: shingle j is
 * units j .. j+n-1 (all m when m < n), words joined by one space, code points as they stand.  Each shingle becomes one
 * 32-bit token, the token hash of its UTF-8 bytes, and the tokens of all documents, with d_tok_offsets, go unchanged to
 * dsk_minhash_bulk_ws.  datasketch_b200/shingle.py:shingles() is the definition in Python.
 * Every count and offset is int64 (the text may exceed 4 GiB); the work is spread over the bytes, not the documents.
 *   dsk_shingle_workspace_size   bytes of the workspace both calls share: 16-byte aligned, owned by the caller, contents
 *                                undefined on entry to dsk_shingle_count; 16 bytes per 2 KiB of text and 28 per document.
 *   dsk_shingle_count  checks the offsets (non-decreasing, inside [0, n_bytes]) and the UTF-8 of every document as CPython's
 *                      strict decoder does, and writes d_doc_status[n_docs + 1] (int32) and d_tok_offsets[n_docs + 1]
 *                      (int64, the exclusive scan of the shingle counts; the total at [n_docs]).  d_doc_status[i] is 0 or
 *                      DSK_SHINGLE_INVALID_UTF8, and such a document gets no shingles; d_doc_status[n_docs] is the OR of
 *                      all of them, plus DSK_SHINGLE_BAD_OFFSETS when the offsets are malformed (then every count is 0 and
 *                      no byte is read through them).  The caller reads the total and the summary back to size d_tokens.
 *   dsk_shingle_hash   with the same text, offsets, unit, n and the workspace dsk_shingle_count filled: writes the token
 *                      of shingle j of document i at d_tokens[d_tok_offsets[i] + j].  hash_kind: 0 = sha1_hash32, or
 *                      DSK_HASH_XXH32 / DSK_HASH_MURMUR3_32 with `seed`. */
#define DSK_SHINGLE_WORD 0
#define DSK_SHINGLE_CHAR 1
#define DSK_SHINGLE_INVALID_UTF8 1
#define DSK_SHINGLE_BAD_OFFSETS 2
DSK_API size_t dsk_shingle_workspace_size(int64_t n_docs, int64_t n_bytes);
DSK_API int dsk_shingle_count(const uint8_t *d_text, const int64_t *d_doc_offsets, int64_t n_docs, int64_t n_bytes, int unit,
                              int n, int64_t *d_tok_offsets, int32_t *d_doc_status, void *d_ws, size_t ws_bytes, void *stream);
DSK_API int dsk_shingle_hash(const uint8_t *d_text, const int64_t *d_doc_offsets, int64_t n_docs, int64_t n_bytes, int unit,
                             int n, int hash_kind, uint32_t seed, const int64_t *d_tok_offsets, uint32_t *d_tokens, void *d_ws,
                             size_t ws_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DSK_H_ */
