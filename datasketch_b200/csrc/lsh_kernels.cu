// lsh_kernels.cu -- device-resident MinHashLSH index (sm_90a).
//
// Replaces the per-document Python work of MinHashLSH._insert / query
// (datasketch/lsh.py:326-347, :370-432 over dict storage, storage.py:209-259):
//   insert: for each band j, bucket[j][ _H(sig[j*r:(j+1)*r]) ].add(doc)
//   query : union over bands of bucket[j][ _H(qsig[j*r:(j+1)*r]) ]
// The reference's bucket key is the r-tuple itself (`_H` = byteswap, lsh.py:537-538), so two
// documents share a bucket iff their r-tuples are EQUAL.  Here a bucket is found through a 64-bit
// fingerprint of the tuple in a per-band open-addressing table (atomicCAS claim), members are
// chained through next[band][doc] (atomicExch on the bucket head), and every candidate is verified
// by comparing the r-tuple itself, so the candidate sets are exactly the reference's.
// A candidate that matches in several bands is emitted once (by the first matching band), which is
// the set-union of lsh.py:426-429.
#include "dsk_common.cuh"

namespace dsk {

// kEmptyKey, lsh_mix64, band_fp: dsk_common.cuh (shared with the signature kernel's fused insert epilogue)

__device__ __forceinline__ bool tuple_eq(const uint32_t *a, const uint32_t *b, int r) {
    bool eq = true;
    for (int q = 0; q < r; ++q) eq = eq && (a[q] == b[q]);
    return eq;
}

// Removal bitmap (dsk_lsh_remove): bit d of removed[d / 32] set = document d was removed since the last compaction.  The
// walks below take it through a template flag RM; the RM = false instantiations never read it and are the kernels that
// ran before removal existed.  Removed documents stay in the bucket chains until dsk_lsh_compact, because they link the
// members behind them: a walk passes through them and never counts, emits, verifies or unites one.
__device__ __forceinline__ bool is_removed(const uint32_t *removed, int64_t d) {
    return (__ldg(removed + (d >> 5)) >> (d & 31)) & 1u;
}

// CTA <-> tile of D = 256 / b new documents.  The tile's rows are contiguous: they are read ONCE with fully coalesced
// loads, each value going to the index's own copy of the signatures (candidates are verified on the r-tuples
// themselves) and to shared memory; then thread <-> (document, band) takes its r-tuple from shared memory for the
// fingerprint and does the table update -- every thread has one atomicCAS chain in flight, which is what hides the DRAM
// latency of the (much larger than L2) tables.  next[] is laid out [doc][band], so the tile's links are one coalesced
// store.  The separate device-to-device copy and the b uncoalesced re-reads of each row of the first version are gone.
__global__ void __launch_bounds__(256) lsh_insert_kernel(const LshDev ix, const uint32_t *__restrict__ new_sig,
                                                         int64_t doc0, int64_t n_new, int docs_per_tile) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_rows, 16);
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    const int64_t n_tiles = (n_new + docs_per_tile - 1) / docs_per_tile;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t i0 = tile * docs_per_tile;
        const int nd = (int)min((int64_t)docs_per_tile, n_new - i0);
        const uint32_t *src = new_sig + i0 * ix.k;
        uint32_t *keep = ix.sig + (doc0 + i0) * ix.k;
        __syncthreads();
        for (int e = threadIdx.x; e < nd * ix.k; e += blockDim.x) {
            const uint32_t v = __ldg(src + e);
            s_rows[e] = v;
            if (keep != src) keep[e] = v;   // (dsk_lsh_insert_tokens' two-kernel route built the rows in place)
        }
        __syncthreads();
        for (int pair = threadIdx.x; pair < nd * ix.b; pair += blockDim.x) {
            const int i = pair / ix.b, band = pair - i * ix.b;
            const int64_t doc = doc0 + i0 + i;
            const uint64_t fp = band_fp(s_rows + i * ix.k + band * ix.r, ix.r, band);
            uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
            uint64_t slot = lsh_mix64(fp) & mask;
            while (true) {
                const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(tab + 2 * slot),
                                                          (unsigned long long)kEmptyKey, (unsigned long long)fp);
                if (prev == kEmptyKey || prev == fp) break;
                slot = (slot + 1) & mask;
            }
            const int32_t old = atomicExch(reinterpret_cast<int32_t *>(tab + 2 * slot + 1), (int32_t)doc);
            ix.next[doc * ix.b + band] = old;
        }
    }
}

// warp <-> query, lane <-> band (bands beyond 32 are handled in further rounds).
// FILL = false: counts[q] = number of distinct candidates.  FILL = true: writes them at out[ptr[q]...].
// RM: removed documents are no candidates.
template <bool FILL, bool RM>
__global__ void __launch_bounds__(256) lsh_query_kernel(const LshDev ix, const uint32_t *__restrict__ qsig, int64_t nq,
                                                        int64_t n_docs, int64_t *__restrict__ counts,
                                                        const int64_t *__restrict__ ptr, int32_t *__restrict__ out,
                                                        const uint32_t *__restrict__ removed) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    for (int64_t q = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < nq; q += warps) {
        const uint32_t *qrow = qsig + q * ix.k;
        int64_t base = FILL ? ptr[q] : 0;
        int64_t total = 0;
        for (int band0 = 0; band0 < ix.b; band0 += 32) {
            const int band = band0 + lane;
            // pass 0 counts this lane's distinct candidates, pass 1 (FILL) writes them after a warp scan
            int mine = 0;
            int64_t wpos = 0;
            for (int pass = 0; pass < (FILL ? 2 : 1); ++pass) {
                int cnt = 0;
                if (band < ix.b) {
                    const uint32_t *qt = qrow + (int64_t)band * ix.r;
                    const uint64_t fp = band_fp(qt, ix.r, band);
                    const uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
                    uint64_t slot = lsh_mix64(fp) & mask;
                    int32_t d = -1;
                    while (true) {
                        const uint64_t kk = tab[2 * slot];
                        if (kk == fp) { d = *reinterpret_cast<const int32_t *>(tab + 2 * slot + 1); break; }
                        if (kk == kEmptyKey) break;
                        slot = (slot + 1) & mask;
                    }
                    while (d >= 0) {
                        if (d < n_docs && !(RM && is_removed(removed, d))) {
                            const uint32_t *drow = ix.sig + (int64_t)d * ix.k;
                            if (tuple_eq(drow + (int64_t)band * ix.r, qt, ix.r)) {
                                bool dup = false;  // already produced by an earlier band?
                                for (int j = 0; j < band && !dup; ++j)
                                    dup = tuple_eq(drow + (int64_t)j * ix.r, qrow + (int64_t)j * ix.r, ix.r);
                                if (!dup) {
                                    if (FILL && pass == 1) out[wpos + cnt] = d;
                                    ++cnt;
                                }
                            }
                        }
                        d = ix.next[(int64_t)d * ix.b + band];
                    }
                }
                if (pass == 0) {
                    mine = cnt;
                    int incl = mine;  // inclusive warp scan of per-lane counts
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                        if (lane >= o) incl += t;
                    }
                    wpos = base + total + (incl - mine);
                    total += __shfl_sync(0xFFFFFFFFu, incl, 31);
                }
            }
        }
        if (!FILL && lane == 0) counts[q] = total;
    }
}

// ---- exclusive scan of int64 counts (three small kernels) -------------------------------------------
constexpr int kScanBlock = 1024;

__global__ void __launch_bounds__(kScanBlock) scan_block_kernel(const int64_t *in, int64_t n, int64_t *out,
                                                                int64_t *block_sums) {
    __shared__ int64_t s[kScanBlock];
    const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
    const int64_t v = i < n ? in[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < kScanBlock; o <<= 1) {
        const int64_t t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
        __syncthreads();
        s[threadIdx.x] += t;
        __syncthreads();
    }
    if (i < n) out[i] = s[threadIdx.x] - v;  // exclusive
    if (threadIdx.x == kScanBlock - 1) block_sums[blockIdx.x] = s[threadIdx.x];
}

__global__ void scan_sums_kernel(int64_t *block_sums, int64_t nb) {  // single thread block, serial over blocks
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int64_t run = 0;
        for (int64_t i = 0; i < nb; ++i) { const int64_t t = block_sums[i]; block_sums[i] = run; run += t; }
        block_sums[nb] = run;
    }
}

__global__ void __launch_bounds__(kScanBlock) scan_add_kernel(int64_t *out, int64_t n, const int64_t *block_sums,
                                                              int64_t nb) {
    const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
    if (i < n) out[i] += block_sums[blockIdx.x];
    if (i == 0) out[n] = block_sums[nb];  // total
}

// ---- launchers ---------------------------------------------------------------------------------------
cudaError_t launch_lsh_insert(const LshDev &ix, const uint32_t *new_sig, int64_t doc0, int64_t n_new, int sm_count,
                              cudaStream_t s) {
    if (n_new <= 0) return cudaSuccess;
    int docs_per_tile = 256 / ix.b;                       // one (document, band) pair per thread
    if (docs_per_tile < 1) docs_per_tile = 1;
    while (docs_per_tile > 1 && (size_t)docs_per_tile * ix.k * 4 > 48 * 1024) --docs_per_tile;
    const size_t smem = (size_t)docs_per_tile * ix.k * 4;
    cudaError_t e = cudaFuncSetAttribute(lsh_insert_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int64_t grid = (n_new + docs_per_tile - 1) / docs_per_tile;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    DSK_LAUNCH(lsh_insert_kernel, (unsigned)grid, 256, smem, s, ix, new_sig, doc0, n_new, docs_per_tile);
    return cudaGetLastError();
}

cudaError_t launch_lsh_query(const LshDev &ix, const uint32_t *qsig, int64_t nq, int64_t n_docs, int64_t *counts,
                             const int64_t *ptr, int32_t *out, int fill, const uint32_t *removed, int sm_count,
                             cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    int64_t grid = (nq + 7) / 8;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    if (removed) {
        if (fill) DSK_LAUNCH((lsh_query_kernel<true, true>), (unsigned)grid, 256, 0, s, ix, qsig, nq, n_docs, counts, ptr, out, removed);
        else DSK_LAUNCH((lsh_query_kernel<false, true>), (unsigned)grid, 256, 0, s, ix, qsig, nq, n_docs, counts, ptr, out, removed);
    } else {
        if (fill) DSK_LAUNCH((lsh_query_kernel<true, false>), (unsigned)grid, 256, 0, s, ix, qsig, nq, n_docs, counts, ptr, out, nullptr);
        else DSK_LAUNCH((lsh_query_kernel<false, false>), (unsigned)grid, 256, 0, s, ix, qsig, nq, n_docs, counts, ptr, out, nullptr);
    }
    return cudaGetLastError();
}

cudaError_t launch_lsh_query(const LshDev &ix, const uint32_t *qsig, int64_t nq, int64_t n_docs, int64_t *counts,
                             const int64_t *ptr, int32_t *out, int fill, int sm_count, cudaStream_t s) {
    return launch_lsh_query(ix, qsig, nq, n_docs, counts, ptr, out, fill, nullptr, sm_count, s);
}

// out has n + 1 entries; scratch needs (n / 1024 + 2) int64
cudaError_t launch_exclusive_scan(const int64_t *in, int64_t n, int64_t *out, int64_t *scratch, cudaStream_t s) {
    const int64_t nb = (n + kScanBlock - 1) / kScanBlock;
    if (n <= 0) return cudaMemsetAsync(out, 0, sizeof(int64_t), s);
    DSK_LAUNCH(scan_block_kernel, (unsigned)nb, kScanBlock, 0, s, in, n, out, scratch);
    DSK_LAUNCH(scan_sums_kernel, 1, 32, 0, s, scratch, nb);
    DSK_LAUNCH(scan_add_kernel, (unsigned)nb, kScanBlock, 0, s, out, n, scratch, nb);
    return cudaGetLastError();
}

}  // namespace dsk

// ---- LSH Forest query (datasketch/lshforest.py:74-128) --------------------------------------------------
// order[tree][pos] = document numbers sorted by (the tree's k-tuple, document number); the sorted list of
// distinct keys + per-key insertion-ordered buckets of the reference flatten to exactly this sequence.
// warp <-> query.  For each prefix length r = k..1: lanes binary-search the l trees in parallel (tuple compare
// on the signatures themselves), then the matches are emitted tree by tree, in sequence order, into the
// query's result list (first `cap` DISTINCT documents), stopping exactly where the reference returns.
namespace dsk {

__device__ __forceinline__ int lex_cmp(const uint32_t *a, const uint32_t *b, int r) {
    for (int q = 0; q < r; ++q) {
        const uint32_t x = a[q], y = b[q];
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

// The warp-held top-k list of the ranked queries (lsh_pairs_kernel's TOPK modes, forest_query_kernel's): lane j holds
// entry j as (best_d, best_eq), -1 / -1 while empty, in the order larger eq, then smaller document number.  Every lane
// calls it with the same candidate c and its count e.  If e >= min_count, c goes in at position popc(ballot(entry j is
// better)): the lanes above it shift up by one shuffle and the lane at it takes c; a candidate that entry topk - 1 beats
// changes nothing.
__device__ __forceinline__ void topk_insert(int32_t &best_d, int32_t &best_eq, int32_t c, int e, int lane, int topk,
                                            int min_count) {
    const bool better = lane < topk && (best_eq > e || (best_eq == e && best_d < c));
    const int at = __popc(__ballot_sync(0xFFFFFFFFu, better));   // entries before c
    if (e >= min_count && at < topk) {
        const int32_t ue = __shfl_up_sync(0xFFFFFFFFu, best_eq, 1);
        const int32_t ud = __shfl_up_sync(0xFFFFFFFFu, best_d, 1);
        if (lane == at) { best_eq = e; best_d = c; }
        else if (lane > at) { best_eq = ue; best_d = ud; }
    }
}

// MODE (FOREST_*, dsk_common.cuh):
//   SET         out_idx[q * cap ...] = the collected list, -1 pads (MinHashLSHForest.query(m, cap)); out_eq, topk and
//               min_count are unused
//   QUERY_TOPK  phase 1 collects the same list of `cap` (= candidates) documents; phase 2 counts each one's eq against
//               the query row over all K words, one document after the other across the warp, and keeps those with
//               eq >= min_count in the warp-held list of topk_insert; lanes < topk store out_idx / out_eq [q * topk + lane]
//   SELF_TOPK   QUERY_TOPK for index row q (the launcher passes qsig = sig, nq = n) with document q skipped while
//               collecting -- by number, so an exact copy of q stays a candidate, and q never counts against cap
// The filter only removes documents from the collected list: which documents are collected does not depend on it.
// SW = words per sample.  SW = 1: MinHash rows, k and r count words.  SW = 2: weighted MinHash rows, sample s = words
// 2s (k, uint32) and 2s + 1 (t, int32 two's complement); K = 2 * sample_size words, and tree t's samples are words
// [2tk, 2(t+1)k).  Compared as unsigned words, these rows sort like the reference's big-endian int64 (k, t) keys (a
// negative t sorts after every non-negative one in both), so the binary search and the emission compare 2r words for
// a prefix of r samples -- never an odd number of words.  eq counts the samples whose two words are both equal, each
// read with one 8-byte load (rows of 2 * sample_size words stay 8-byte aligned).
template <int MODE, int SW>
__global__ void __launch_bounds__(128) forest_query_kernel(const uint32_t *__restrict__ sig,
                                                           const int32_t *__restrict__ order, int64_t n, int K, int l,
                                                           int k, const uint32_t *__restrict__ qsig, int64_t nq,
                                                           int cap, int32_t *__restrict__ out_idx,
                                                           int32_t *__restrict__ out_eq, int topk, int min_count) {
    DSK_DYNAMIC_SMEM_T(int32_t, s_res, 4);  // [warps][cap]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int32_t *res = s_res + warp * cap;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t q = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; q < nq; q += warps) {
        const uint32_t *qrow = qsig + q * K;
        int cnt = 0;
        bool done = false;
        for (int r = k; r >= 1 && !done; --r) {
            for (int t0 = 0; t0 < l && !done; t0 += 32) {
                const int tree = t0 + lane;
                int64_t lo = 0;
                if (tree < l) {  // lower bound of the r-prefix in this lane's tree
                    const uint32_t *qt = qrow + tree * SW * k;
                    const int32_t *ord = order + (int64_t)tree * n;
                    int64_t hi = n;
                    while (lo < hi) {
                        const int64_t mid = lo + ((hi - lo) >> 1);
                        if (lex_cmp(sig + (int64_t)ord[mid] * K + tree * SW * k, qt, SW * r) < 0) lo = mid + 1;
                        else hi = mid;
                    }
                }
                const int ntree = min(32, l - t0);
                for (int j = 0; j < ntree && !done; ++j) {  // emit in tree order; lane 0 owns the result list
                    int64_t pos = __shfl_sync(0xFFFFFFFFu, lo, j);
                    if (lane == 0) {
                        const int tj = t0 + j;
                        const uint32_t *qt = qrow + tj * SW * k;
                        const int32_t *ord = order + (int64_t)tj * n;
                        while (pos < n) {
                            const int32_t d = ord[pos];
                            if (lex_cmp(sig + (int64_t)d * K + tj * SW * k, qt, SW * r) != 0) break;
                            bool seen = MODE == FOREST_SELF_TOPK && d == q;
                            for (int e = 0; e < cnt; ++e) seen = seen || (res[e] == d);
                            if (!seen) {
                                res[cnt++] = d;
                                if (cnt >= cap) break;
                            }
                            ++pos;
                        }
                    }
                    cnt = __shfl_sync(0xFFFFFFFFu, cnt, 0);
                    done = cnt >= cap;
                }
            }
        }
        __syncwarp();
        if constexpr (MODE == FOREST_SET) {
            for (int e = lane; e < cap; e += 32) out_idx[q * cap + e] = e < cnt ? res[e] : -1;
        } else {
            int32_t best_d = -1, best_eq = -1;   // entry `lane` of the ranked list
            for (int e = 0; e < cnt; ++e) {
                const int32_t c = res[e];
                const uint32_t *crow = sig + (int64_t)c * K;
                int m = 0;
                if constexpr (SW == 1) {
                    for (int w = lane; w < K; w += 32) m += crow[w] == qrow[w];
                } else {
                    // a sample's two words as one 64-bit value: equal iff k and t are both equal
                    const uint64_t *c2 = reinterpret_cast<const uint64_t *>(crow);
                    const uint64_t *q2 = reinterpret_cast<const uint64_t *>(qrow);
                    for (int w = lane; w < (K >> 1); w += 32) m += c2[w] == q2[w];
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xFFFFFFFFu, m, o);
                topk_insert(best_d, best_eq, c, m, lane, topk, min_count);
            }
            if (lane < topk) { out_idx[q * topk + lane] = best_d; out_eq[q * topk + lane] = best_eq; }
        }
        __syncwarp();
    }
}

template <int MODE, int SW>
static cudaError_t forest_launch_t(const uint32_t *sig, const int32_t *order, int64_t n, int K, int l, int k,
                                   const uint32_t *qsig, int64_t nq, int cap, int32_t *idx, int32_t *eq, int topk,
                                   int min_count, int sm_count, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    int64_t grid = (nq + 3) / 4;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    const size_t smem = (size_t)4 * cap * sizeof(int32_t);
    DSK_LAUNCH((forest_query_kernel<MODE, SW>), (unsigned)grid, 128, smem, s, sig, order, n, K, l, k, qsig, nq, cap, idx,
               eq, topk, min_count);
    return cudaGetLastError();
}

cudaError_t launch_forest(int mode, int sw, const uint32_t *sig, const int32_t *order, int64_t n, int K, int l, int k,
                          const uint32_t *qsig, int64_t nq, int cap, int32_t *idx, int32_t *eq, int topk, int min_count,
                          int sm_count, cudaStream_t s) {
    if (mode == FOREST_SELF_TOPK) { qsig = sig; nq = n; }
#define DSK_FOREST_CASE(M)                                                                                                  \
    if (mode == M)                                                                                                          \
        return sw == 2 ? forest_launch_t<M, 2>(sig, order, n, K, l, k, qsig, nq, cap, idx, eq, topk, min_count, sm_count, s) \
                       : forest_launch_t<M, 1>(sig, order, n, K, l, k, qsig, nq, cap, idx, eq, topk, min_count, sm_count, s);
    DSK_FOREST_CASE(FOREST_SET)
    DSK_FOREST_CASE(FOREST_QUERY_TOPK)
    DSK_FOREST_CASE(FOREST_SELF_TOPK)
#undef DSK_FOREST_CASE
    return cudaErrorInvalidValue;
}

cudaError_t launch_forest_query(const uint32_t *sig, const int32_t *order, int64_t n, int K, int l, int k,
                                const uint32_t *qsig, int64_t nq, int topk, int32_t *out, int sm_count,
                                cudaStream_t s) {
    return launch_forest(FOREST_SET, 1, sig, order, n, K, l, k, qsig, nq, topk, out, nullptr, 0, 0, sm_count, s);
}

}  // namespace dsk

// ---- self-join of the index: candidate pairs and duplicate clusters ----------------------------------------------------
// Documents i and d (d < i) are a candidate pair iff some band's r-tuples are equal -- d is in MinHashLSH.query(row i),
// lsh.py:370-432 -- and eq(i, d), the number of the K positions where the rows agree (MinHash.jaccard * K,
// minhash.py:324), is at least min_count.  Clusters are the connected components of that pair graph, each labelled by its
// smallest document number.
namespace dsk {

// Loads and stores of union-find parents that race with hooks are relaxed (ld_relaxed / st_relaxed, dsk_common.cuh).

// Lock-free union-find on parent[] with parent[x] <= x at all times.  A hook replaces a root's self-link by a SMALLER
// root (atomicCAS, so it fails if the root was hooked meanwhile), so every path strictly decreases and the root of each
// tree is its smallest member.  Path halving may store any ancestor of a non-root x: ancestors never stop being ones.
__device__ __forceinline__ int32_t uf_find(int32_t *parent, int32_t x) {
    while (true) {
        const int32_t p = ld_relaxed(parent + x);
        if (p == x) return x;
        const int32_t g = ld_relaxed(parent + p);
        if (g != p) st_relaxed(parent + x, g);
        x = g;
    }
}

__device__ __forceinline__ void uf_union(int32_t *parent, int32_t a, int32_t b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        const int32_t hi = a > b ? a : b, lo = a > b ? b : a;
        if (atomicCAS(parent + hi, hi, lo) == hi) return;
        a = hi;   // hi was hooked by another thread in between: find both roots again
        b = lo;
    }
}

__global__ void __launch_bounds__(256) uf_init_kernel(int32_t *labels, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        labels[i] = (int32_t)i;
}

// RM: a removed document gets the label -1.  Nothing ever hooks a removed document (the walks never unite one), so it is
// a root of its own that no other document's path passes through, and its plain store races with no find.
template <bool RM>
__global__ void __launch_bounds__(256) uf_flatten_kernel(int32_t *labels, int64_t n, const uint32_t *__restrict__ removed) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (RM && is_removed(removed, i)) labels[i] = -1;
        else st_relaxed(labels + i, uf_find(labels, (int32_t)i));
    }
}

enum { PAIRS_COUNT = 0, PAIRS_FILL = 1, PAIRS_UNION = 2, QUERY_COUNT = 3, QUERY_FILL = 4, QUERY_BEST = 5, QUERY_TOPK = 6,
       SELF_TOPK = 7 };

// warp <-> document i, lane <-> band (bands beyond 32 in further rounds), row i staged once in shared memory.  Each lane
// probes its band's table with the fingerprint of i's own tuple and walks the bucket's chain to its next partner d: d < i,
// the tuple really equal, and no earlier band with equal tuples (the first matching band emits the pair, as in
// lsh_query_kernel).  Then the warp counts eq for every lane's pending partner together -- 32 lanes over the two K-word
// rows and a shuffle reduction, one partner after the other -- and the partners with eq >= min_count are kept:
//   PAIRS_COUNT  counts[i] = number kept
//   PAIRS_FILL   written at idx / eq [ptr[i] ...), in no particular order
//   PAIRS_UNION  united with i in labels[] (nothing materialised)
// RM: a removed i has no partners (its whole iteration is skipped, warp-uniformly; PAIRS_COUNT still writes counts[i] = 0),
// and a removed d is no partner.
// The QUERY modes run the same walk for the nq rows of qsig, which are not in the index: row i is qsig + i * k, and every
// document d < n_docs is eligible (the bound of lsh_query_kernel), so the partners of query i are exactly query(row i):
//   QUERY_COUNT  counts[i] = number kept
//   QUERY_FILL   written at idx / eq [ptr[i] ...), in no particular order
//   QUERY_BEST   idx[i] / eq[i] = the kept partner with the largest eq, the smallest d among equal ones (-1 / -1: none).
//                Each lane keeps its own best and a warp shuffle reduction picks the query's: no atomics.
// The TOPK modes keep the first `topk` (<= 32) kept partners in the order larger eq, then smaller d: lane j holds entry j,
// -1 / -1 while empty.  Every candidate's eq is counted, and right after the count (where every lane knows the candidate and
// its eq) a kept one is inserted at position popc(ballot(entry j is better)): the lanes above it shift up by one shuffle,
// the lane at it takes the new entry, and a candidate that entry topk - 1 beats changes nothing.  At the end of the row
// lanes < topk store idx / eq [i * topk + lane].  No shared-memory list and no atomics.
//   QUERY_TOPK   the query walk (row i = qsig + i * k, every d < n_docs)
//   SELF_TOPK    index row i against every document d < n_docs with d != i: i's nearest neighbours; with RM a removed i
//                stores a row of -1 and skips its walk, warp-uniformly
// In the PAIRS modes qsig and nq are unused and the code is the self-join's alone; only the TOPK modes read topk.
// SW = words per sample.  SW = 1: MinHash rows, eq counts equal words.  SW = 2: weighted MinHash rows, sample s = words
// 2s (k) and 2s + 1 (t), ix.k = 2 * sample_size and ix.r = 2 * r words; eq counts the samples whose two words are both
// equal (WeightedMinHash.jaccard * sample_size), each read with one 8-byte load (rows of 2 * sample_size words stay 8-byte
// aligned).  Bands, chains, tuple checks and the first-matching-band rule work on words and need no change.
template <int MODE, bool RM, int SW = 1>
__global__ void __launch_bounds__(256) lsh_pairs_kernel(const LshDev ix, int64_t n_docs, int min_count,
                                                        int64_t *__restrict__ counts, const int64_t *__restrict__ ptr,
                                                        int32_t *__restrict__ out_idx, int32_t *__restrict__ out_eq,
                                                        int32_t *labels, const uint32_t *__restrict__ removed,
                                                        const uint32_t *__restrict__ qsig, int64_t nq, int topk) {
    constexpr bool QUERY = MODE >= QUERY_COUNT && MODE != SELF_TOPK;
    constexpr bool TOPK = MODE == QUERY_TOPK || MODE == SELF_TOPK;
    DSK_DYNAMIC_SMEM_T(uint32_t, s_rows, 16);   // [warps][k]
    const int lane = threadIdx.x & 31;
    uint32_t *row = s_rows + (int64_t)(threadIdx.x >> 5) * ix.k;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    const bool need_eq = MODE == PAIRS_FILL || MODE == QUERY_FILL || MODE == QUERY_BEST || TOPK || min_count > 0;
    const unsigned below = (1u << lane) - 1u;
    for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < (QUERY ? nq : n_docs); i += warps) {
        if (!QUERY && RM && is_removed(removed, i)) {
            if (MODE == PAIRS_COUNT && lane == 0) counts[i] = 0;
            if (MODE == SELF_TOPK && lane < topk) { out_idx[i * topk + lane] = -1; out_eq[i * topk + lane] = -1; }
            continue;
        }
        const int64_t bound = QUERY || MODE == SELF_TOPK ? n_docs : i;   // partners d < bound (SELF_TOPK: and d != i)
        int32_t best_d = -1, best_eq = -1;          // QUERY_BEST: this lane's best kept partner; TOPK: entry `lane`
        const uint32_t *irow = (QUERY ? qsig : ix.sig) + i * ix.k;
        __syncwarp();
        for (int w = lane; w < ix.k; w += 32) row[w] = irow[w];
        __syncwarp();
        int64_t total = 0;   // partners kept so far (the same in every lane)
        for (int band0 = 0; band0 < ix.b; band0 += 32) {
            const int band = band0 + lane;
            const uint32_t *it = row + band * ix.r;
            int32_t d = -1;
            if (band < ix.b) {
                const uint64_t fp = band_fp(it, ix.r, band);
                const uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
                uint64_t slot = lsh_mix64(fp) & mask;
                while (true) {
                    const uint64_t kk = tab[2 * slot];
                    if (kk == fp) { d = *reinterpret_cast<const int32_t *>(tab + 2 * slot + 1); break; }
                    if (kk == kEmptyKey) break;
                    slot = (slot + 1) & mask;
                }
            }
            while (true) {
                int32_t cand = -1;
                while (d >= 0) {
                    const int32_t cur = d;
                    d = ix.next[(int64_t)cur * ix.b + band];
                    if (cur < bound && !(MODE == SELF_TOPK && cur == i) && !(RM && is_removed(removed, cur))) {
                        const uint32_t *drow = ix.sig + (int64_t)cur * ix.k;
                        if (tuple_eq(drow + band * ix.r, it, ix.r)) {
                            bool dup = false;
                            for (int j = 0; j < band && !dup; ++j)
                                dup = tuple_eq(drow + j * ix.r, row + j * ix.r, ix.r);
                            if (!dup) { cand = cur; break; }
                        }
                    }
                }
                const unsigned pending = __ballot_sync(0xFFFFFFFFu, cand >= 0);
                if (pending == 0u) break;
                int eq = 0;
                if (need_eq) {
                    for (unsigned m = pending; m; m &= m - 1u) {
                        const int src = __ffs(m) - 1;
                        const uint32_t *crow = ix.sig + (int64_t)__shfl_sync(0xFFFFFFFFu, cand, src) * ix.k;
                        int e = 0;
                        if constexpr (SW == 1) {
                            for (int w = lane; w < ix.k; w += 32) e += crow[w] == row[w];
                        } else {
                            // a sample's two words as one 64-bit value: equal iff k and t are both equal
                            const uint64_t *c2 = reinterpret_cast<const uint64_t *>(crow);
                            const uint64_t *r2 = reinterpret_cast<const uint64_t *>(row);
                            for (int w = lane; w < (ix.k >> 1); w += 32) e += c2[w] == r2[w];
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xFFFFFFFFu, e, o);
                        if (lane == src) eq = e;
                        if constexpr (TOPK) {   // e and c are the same in every lane: the insert is warp-uniform
                            const int32_t c = __shfl_sync(0xFFFFFFFFu, cand, src);
                            topk_insert(best_d, best_eq, c, e, lane, topk, min_count);
                        }
                    }
                }
                const bool keep = cand >= 0 && eq >= min_count;
                if (MODE == PAIRS_UNION) {
                    if (keep) uf_union(labels, (int32_t)i, cand);
                } else if (MODE == QUERY_BEST) {
                    if (keep && (eq > best_eq || (eq == best_eq && cand < best_d))) { best_eq = eq; best_d = cand; }
                } else if (TOPK) {
                    // inserted above, in the eq loop
                } else {
                    const unsigned kept = __ballot_sync(0xFFFFFFFFu, keep);
                    if ((MODE == PAIRS_FILL || MODE == QUERY_FILL) && keep) {
                        const int64_t pos = ptr[i] + total + __popc(kept & below);
                        out_idx[pos] = cand;
                        out_eq[pos] = eq;
                    }
                    total += __popc(kept);
                }
            }
        }
        if ((MODE == PAIRS_COUNT || MODE == QUERY_COUNT) && lane == 0) counts[i] = total;
        if (MODE == QUERY_BEST) {   // largest eq, then smallest d; a lane without a kept partner holds (-1, -1) and loses
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const int32_t oe = __shfl_xor_sync(0xFFFFFFFFu, best_eq, o), od = __shfl_xor_sync(0xFFFFFFFFu, best_d, o);
                if (oe > best_eq || (oe == best_eq && od < best_d)) { best_eq = oe; best_d = od; }
            }
            if (lane == 0) { out_idx[i] = best_d; out_eq[i] = best_eq; }
        }
        if (TOPK && lane < topk) { out_idx[i * topk + lane] = best_d; out_eq[i * topk + lane] = best_eq; }
    }
}

// min_count = 0: thread <-> (document i, band).  i is united with the FIRST other member of its band's chain whose tuple
// equals i's, so the members with one tuple form a star around the first of them in chain order -- the components of the
// full clique, in time linear in the index (plus the members of other tuples that share the chain's fingerprint).
// RM: a removed i does nothing, and a remaining i is united with the first OTHER REMAINING member with its tuple.  The
// star argument holds for the remaining members alone: let f be the first remaining member with the tuple in chain order;
// every other remaining member with the tuple meets f first and unites with it, and f unites with the second one.  So
// the remaining members with one tuple are connected, and no removed document is ever united.
template <bool RM>
__global__ void __launch_bounds__(256) lsh_link_kernel(const LshDev ix, int64_t n_docs, int32_t *labels,
                                                       const uint32_t *__restrict__ removed) {
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    const int64_t n_pairs = n_docs * ix.b;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pairs; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = p / ix.b;
        if (RM && is_removed(removed, i)) continue;
        const int band = (int)(p - i * ix.b);
        const uint32_t *it = ix.sig + i * ix.k + band * ix.r;
        const uint64_t fp = band_fp(it, ix.r, band);
        const uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
        uint64_t slot = lsh_mix64(fp) & mask;
        int32_t d = -1;
        while (true) {
            const uint64_t kk = tab[2 * slot];
            if (kk == fp) { d = *reinterpret_cast<const int32_t *>(tab + 2 * slot + 1); break; }
            if (kk == kEmptyKey) break;
            slot = (slot + 1) & mask;
        }
        while (d >= 0) {
            if (d != i && !(RM && is_removed(removed, d)) && tuple_eq(ix.sig + (int64_t)d * ix.k + band * ix.r, it, ix.r)) {
                uf_union(labels, (int32_t)i, d);
                break;
            }
            d = ix.next[(int64_t)d * ix.b + band];
        }
    }
}

// the pair walk's launch shape for `rows` staged rows (documents, or queries with M0 = QUERY_COUNT): up to 8 warps per
// CTA, each with a K-word row in shared memory.  Allows that much shared memory to the modes M0, M0 + 1 and M0 + 2.
template <bool RM, int M0 = PAIRS_COUNT, int SW = 1>
static cudaError_t pairs_shape(const LshDev &ix, int64_t rows, int sm_count, int *warps, unsigned *grid, size_t *smem) {
    int w = 8;
    while (w > 1 && (size_t)w * ix.k * 4 > 48 * 1024) w >>= 1;
    *warps = w;
    *smem = (size_t)w * ix.k * 4;
    int64_t g = (rows + w - 1) / w;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    *grid = (unsigned)g;
    cudaError_t e = cudaFuncSetAttribute(lsh_pairs_kernel<M0, RM, SW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(lsh_pairs_kernel<M0 + 1, RM, SW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(lsh_pairs_kernel<M0 + 2, RM, SW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
    return e;
}

template <bool RM, int SW>
static cudaError_t launch_pairs_t(const LshDev &ix, int64_t n_docs, int min_count, int64_t *counts, const int64_t *ptr,
                                  int32_t *idx, int32_t *eq, const uint32_t *removed, int sm_count, cudaStream_t s) {
    int warps;
    unsigned grid;
    size_t smem;
    cudaError_t e = pairs_shape<RM, PAIRS_COUNT, SW>(ix, n_docs, sm_count, &warps, &grid, &smem);
    if (e != cudaSuccess) return e;
    if (counts)
        DSK_LAUNCH((lsh_pairs_kernel<PAIRS_COUNT, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, counts, nullptr,
                   nullptr, nullptr, nullptr, removed, nullptr, 0, 0);
    else
        DSK_LAUNCH((lsh_pairs_kernel<PAIRS_FILL, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, ptr, idx, eq,
                   nullptr, removed, nullptr, 0, 0);
    return cudaGetLastError();
}

// counts != nullptr: counts[i] for every document; else the fill of idx / eq at ptr[i].  removed != nullptr: the
// removal-aware walk.  sw: words per sample of the index's rows (1 or 2).
cudaError_t launch_lsh_pairs(const LshDev &ix, int sw, int64_t n_docs, int min_count, int64_t *counts, const int64_t *ptr,
                             int32_t *idx, int32_t *eq, const uint32_t *removed, int sm_count, cudaStream_t s) {
    if (n_docs <= 0) return cudaSuccess;
    if (sw == 2) {
        if (removed) return launch_pairs_t<true, 2>(ix, n_docs, min_count, counts, ptr, idx, eq, removed, sm_count, s);
        return launch_pairs_t<false, 2>(ix, n_docs, min_count, counts, ptr, idx, eq, nullptr, sm_count, s);
    }
    if (removed) return launch_pairs_t<true, 1>(ix, n_docs, min_count, counts, ptr, idx, eq, removed, sm_count, s);
    return launch_pairs_t<false, 1>(ix, n_docs, min_count, counts, ptr, idx, eq, nullptr, sm_count, s);
}

template <bool RM, int SW>
static cudaError_t launch_clusters_t(const LshDev &ix, int64_t n_docs, int min_count, int32_t *labels,
                                     const uint32_t *removed, int sm_count, cudaStream_t s) {
    int64_t grid = (n_docs + 255) / 256;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    DSK_LAUNCH(uf_init_kernel, (unsigned)grid, 256, 0, s, labels, n_docs);
    if (min_count == 0) {
        int64_t lg = (n_docs * ix.b + 255) / 256;
        if (lg > (int64_t)sm_count * 8) lg = (int64_t)sm_count * 8;
        DSK_LAUNCH(lsh_link_kernel<RM>, (unsigned)lg, 256, 0, s, ix, n_docs, labels, removed);
    } else {
        int warps;
        unsigned pg;
        size_t smem;
        cudaError_t e = pairs_shape<RM, PAIRS_COUNT, SW>(ix, n_docs, sm_count, &warps, &pg, &smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH((lsh_pairs_kernel<PAIRS_UNION, RM, SW>), pg, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, nullptr,
                   nullptr, nullptr, labels, removed, nullptr, 0, 0);
    }
    DSK_LAUNCH(uf_flatten_kernel<RM>, (unsigned)grid, 256, 0, s, labels, n_docs, removed);
    return cudaGetLastError();
}

cudaError_t launch_lsh_clusters(const LshDev &ix, int sw, int64_t n_docs, int min_count, int32_t *labels,
                                const uint32_t *removed, int sm_count, cudaStream_t s) {
    if (n_docs <= 0) return cudaSuccess;
    if (sw == 2) {
        if (removed) return launch_clusters_t<true, 2>(ix, n_docs, min_count, labels, removed, sm_count, s);
        return launch_clusters_t<false, 2>(ix, n_docs, min_count, labels, nullptr, sm_count, s);
    }
    if (removed) return launch_clusters_t<true, 1>(ix, n_docs, min_count, labels, removed, sm_count, s);
    return launch_clusters_t<false, 1>(ix, n_docs, min_count, labels, nullptr, sm_count, s);
}

template <bool RM, int SW>
static cudaError_t launch_query_pairs_t(const LshDev &ix, const uint32_t *qsig, int64_t nq, int64_t n_docs, int min_count,
                                        int mode, int64_t *counts, const int64_t *ptr, int32_t *idx, int32_t *eq,
                                        const uint32_t *removed, int sm_count, cudaStream_t s) {
    int warps;
    unsigned grid;
    size_t smem;
    cudaError_t e = pairs_shape<RM, QUERY_COUNT, SW>(ix, nq, sm_count, &warps, &grid, &smem);
    if (e != cudaSuccess) return e;
    if (mode == QUERY_COUNT)
        DSK_LAUNCH((lsh_pairs_kernel<QUERY_COUNT, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, counts, nullptr,
                   nullptr, nullptr, nullptr, removed, qsig, nq, 0);
    else if (mode == QUERY_FILL)
        DSK_LAUNCH((lsh_pairs_kernel<QUERY_FILL, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, ptr, idx, eq,
                   nullptr, removed, qsig, nq, 0);
    else
        DSK_LAUNCH((lsh_pairs_kernel<QUERY_BEST, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, nullptr, idx,
                   eq, nullptr, removed, qsig, nq, 0);
    return cudaGetLastError();
}

// The pair walk for the nq rows of qsig against the index's first n_docs documents.  counts != nullptr: counts[q] of the
// kept candidates; ptr != nullptr: the fill of idx / eq at ptr[q]; else idx[q] / eq[q] = q's best kept candidate.
cudaError_t launch_lsh_query_pairs(const LshDev &ix, int sw, const uint32_t *qsig, int64_t nq, int64_t n_docs, int min_count,
                                   int64_t *counts, const int64_t *ptr, int32_t *idx, int32_t *eq, const uint32_t *removed,
                                   int sm_count, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    const int mode = counts ? QUERY_COUNT : ptr ? QUERY_FILL : QUERY_BEST;
    if (sw == 2) {
        if (removed)
            return launch_query_pairs_t<true, 2>(ix, qsig, nq, n_docs, min_count, mode, counts, ptr, idx, eq, removed, sm_count, s);
        return launch_query_pairs_t<false, 2>(ix, qsig, nq, n_docs, min_count, mode, counts, ptr, idx, eq, nullptr, sm_count, s);
    }
    if (removed) return launch_query_pairs_t<true, 1>(ix, qsig, nq, n_docs, min_count, mode, counts, ptr, idx, eq, removed, sm_count, s);
    return launch_query_pairs_t<false, 1>(ix, qsig, nq, n_docs, min_count, mode, counts, ptr, idx, eq, nullptr, sm_count, s);
}

template <bool RM, int SW>
static cudaError_t launch_topk_t(const LshDev &ix, const uint32_t *qsig, int64_t nq, int64_t n_docs, int min_count, int k,
                                 int32_t *idx, int32_t *eq, const uint32_t *removed, int sm_count, cudaStream_t s) {
    const int64_t rows = qsig ? nq : n_docs;
    int warps;
    unsigned grid;
    size_t smem;
    cudaError_t e = pairs_shape<RM, QUERY_BEST, SW>(ix, rows, sm_count, &warps, &grid, &smem);   // QUERY_BEST, both TOPK
    if (e != cudaSuccess) return e;
    if (qsig)
        DSK_LAUNCH((lsh_pairs_kernel<QUERY_TOPK, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, nullptr, idx,
                   eq, nullptr, removed, qsig, nq, k);
    else
        DSK_LAUNCH((lsh_pairs_kernel<SELF_TOPK, RM, SW>), grid, 32 * warps, smem, s, ix, n_docs, min_count, nullptr, nullptr, idx,
                   eq, nullptr, removed, nullptr, 0, k);
    return cudaGetLastError();
}

// Each row's first k (1..32) kept partners, larger eq first, then smaller d, -1 / -1 behind them, at idx / eq [row * k ...):
// qsig != nullptr: the nq query rows against the first n_docs documents; qsig == nullptr: the n_docs documents' own rows,
// each against every other document (its nearest neighbours).
cudaError_t launch_lsh_topk(const LshDev &ix, int sw, const uint32_t *qsig, int64_t nq, int64_t n_docs, int min_count, int k,
                            int32_t *idx, int32_t *eq, const uint32_t *removed, int sm_count, cudaStream_t s) {
    if ((qsig ? nq : n_docs) <= 0) return cudaSuccess;
    if (sw == 2) {
        if (removed) return launch_topk_t<true, 2>(ix, qsig, nq, n_docs, min_count, k, idx, eq, removed, sm_count, s);
        return launch_topk_t<false, 2>(ix, qsig, nq, n_docs, min_count, k, idx, eq, nullptr, sm_count, s);
    }
    if (removed) return launch_topk_t<true, 1>(ix, qsig, nq, n_docs, min_count, k, idx, eq, removed, sm_count, s);
    return launch_topk_t<false, 1>(ix, qsig, nq, n_docs, min_count, k, idx, eq, nullptr, sm_count, s);
}

}  // namespace dsk

// ---- removal and compaction ---------------------------------------------------------------------------------------------
// MinHashLSH.remove (lsh.py:509-528) drops a key from its buckets.  Here a removal only sets the document's bit in the
// handle's bitmap (cap_docs bits, 1.25 MB at 10M documents: L2-resident), and the walks above skip it.  Compaction then
// renumbers the remaining documents 0..m-1 in their old order, moves their rows down inside the index's own storage and
// rebuilds the bucket tables from them, which gives the capacity back.
namespace dsk {

#ifdef DSK_EMU
inline void atomic_add_i64(int64_t *p, int64_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
#else
__device__ __forceinline__ void atomic_add_i64(int64_t *p, int64_t v) {
    atomicAdd(reinterpret_cast<unsigned long long *>(p), (unsigned long long)v);
}
#endif

// thread <-> listed id.  status[0] += ids outside [0, n_docs), status[1] += ids whose bit was set already (a repeat within
// docs counts once: one of the atomicOr's sees the bit clear).  The loop runs over whole warps, so that every lane takes part
// in the ballots that aggregate the counts before lane 0's atomicAdd.
__global__ void __launch_bounds__(256) lsh_remove_kernel(uint32_t *removed, const int32_t *__restrict__ docs, int64_t n,
                                                         int64_t n_docs, int64_t *status) {
    const int lane = threadIdx.x & 31;
    const int64_t n_up = (n + 31) & ~(int64_t)31;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_up; j += (int64_t)gridDim.x * blockDim.x) {
        bool bad = false, again = false;
        if (j < n) {
            const int32_t d = docs[j];
            if (d < 0 || d >= n_docs) {
                bad = true;
            } else {
                const uint32_t bit = 1u << (d & 31);
                again = (atomicOr(removed + (d >> 5), bit) & bit) != 0u;
            }
        }
        const unsigned nb = __ballot_sync(0xFFFFFFFFu, bad), na = __ballot_sync(0xFFFFFFFFu, again);
        if (lane == 0 && nb) atomic_add_i64(status, __popc(nb));
        if (lane == 0 && na) atomic_add_i64(status + 1, __popc(na));
    }
}

// out[j] = 1 iff docs[j] is in [0, n_docs) and not removed (removed == nullptr: nothing was)
__global__ void __launch_bounds__(256) lsh_alive_kernel(const uint32_t *__restrict__ removed, const int32_t *__restrict__ docs,
                                                        int64_t n, int64_t n_docs, uint8_t *__restrict__ out) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        const int32_t d = docs[j];
        out[j] = d >= 0 && d < n_docs && !(removed && is_removed(removed, d));
    }
}

// surviving bits of bitmap word w among documents 0..n_docs-1
__device__ __forceinline__ uint32_t alive_bits(const uint32_t *removed, int64_t w, int64_t n_docs) {
    const int64_t left = n_docs - w * 32;
    const uint32_t valid = left >= 32 ? 0xFFFFFFFFu : (1u << left) - 1u;
    return ~removed[w] & valid;
}

__global__ void __launch_bounds__(256) compact_count_kernel(const uint32_t *__restrict__ removed, int64_t n_words,
                                                            int64_t n_docs, int64_t *__restrict__ word_cnt) {
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x)
        word_cnt[w] = __popc(alive_bits(removed, w, n_docs));
}

// remap[i] = new number of i (word prefix + surviving bits below i), -1 if removed; new2old[remap[i]] = i
__global__ void __launch_bounds__(256) compact_remap_kernel(const uint32_t *__restrict__ removed, int64_t n_docs,
                                                            const int64_t *__restrict__ word_ptr, int32_t *__restrict__ remap,
                                                            int32_t *__restrict__ new2old) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_docs; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t w = i >> 5;
        const int bit = (int)(i & 31);
        const uint32_t alive = alive_bits(removed, w, n_docs);
        if ((alive >> bit) & 1u) {
            const int32_t t = (int32_t)(word_ptr[w] + __popc(alive & ((1u << bit) - 1u)));
            remap[i] = t;
            new2old[t] = (int32_t)i;
        } else {
            remap[i] = -1;
        }
    }
}

// warp <-> new number t in [a, b): stage[(t - a) * k ...] = row new2old[t]
__global__ void __launch_bounds__(256) compact_gather_kernel(const uint32_t *__restrict__ sig, int k,
                                                             const int32_t *__restrict__ new2old, int64_t a, int64_t b,
                                                             uint32_t *__restrict__ stage) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t t = a + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < b; t += warps) {
        const uint32_t *src = sig + (int64_t)new2old[t] * k;
        uint32_t *dst = stage + (t - a) * k;
        for (int w = lane; w < k; w += 32) dst[w] = src[w];
    }
}

constexpr size_t kCompactStageBytes = (size_t)64 << 20;   // rows moved per chunk of the compaction

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static int64_t compact_stage_rows(int64_t n_docs, int k) {
    int64_t rows = (int64_t)(kCompactStageBytes / ((size_t)k * 4));
    if (rows < 1) rows = 1;
    return rows < n_docs ? rows : n_docs;
}

// word counts int64[n_words] | word prefix int64[n_words + 1] | scan scratch int64[n_words / 1024 + 2] | new -> old
// int32[n_docs] | row staging (at most kCompactStageBytes): nothing that grows as n_docs * k
size_t lsh_compact_workspace_bytes(int64_t n_docs, int k) {
    if (n_docs <= 0) return 0;
    const int64_t n_words = (n_docs + 31) / 32;
    return align256(n_words * 8) + align256((n_words + 1) * 8) + align256((n_words / 1024 + 2) * 8) +
           align256((size_t)n_docs * 4) + align256((size_t)compact_stage_rows(n_docs, k) * k * 4);
}

cudaError_t launch_lsh_remove(uint32_t *removed, const int32_t *docs, int64_t n, int64_t n_docs, int64_t *status,
                              int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    int64_t grid = (n + 255) / 256;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    DSK_LAUNCH(lsh_remove_kernel, (unsigned)grid, 256, 0, s, removed, docs, n, n_docs, status);
    return cudaGetLastError();
}

cudaError_t launch_lsh_alive(const uint32_t *removed, const int32_t *docs, int64_t n, int64_t n_docs, uint8_t *out,
                             int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    int64_t grid = (n + 255) / 256;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    DSK_LAUNCH(lsh_alive_kernel, (unsigned)grid, 256, 0, s, removed, docs, n, n_docs, out);
    return cudaGetLastError();
}

cudaError_t launch_lsh_identity(int32_t *remap, int64_t n, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    int64_t grid = (n + 255) / 256;
    if (grid > (int64_t)sm_count * 8) grid = (int64_t)sm_count * 8;
    DSK_LAUNCH(uf_init_kernel, (unsigned)grid, 256, 0, s, remap, n);
    return cudaGetLastError();
}

// Compacts the first n_docs documents of ix by the bitmap `removed`: remap[i] = new number or -1, *m = the number of
// remaining documents.  Synchronises s once, to read m.  The caller then clears the bitmap and sets its n_docs to m.
cudaError_t lsh_compact(const LshDev &ix, const uint32_t *removed, int64_t n_docs, int32_t *remap, void *ws, int64_t *m,
                        int sm_count, cudaStream_t s) {
    const int64_t n_words = (n_docs + 31) / 32;
    char *p = static_cast<char *>(ws);
    int64_t *word_cnt = reinterpret_cast<int64_t *>(p);
    p += align256(n_words * 8);
    int64_t *word_ptr = reinterpret_cast<int64_t *>(p);
    p += align256((n_words + 1) * 8);
    int64_t *scratch = reinterpret_cast<int64_t *>(p);
    p += align256((n_words / 1024 + 2) * 8);
    int32_t *new2old = reinterpret_cast<int32_t *>(p);
    p += align256((size_t)n_docs * 4);
    uint32_t *stage = reinterpret_cast<uint32_t *>(p);
    const int64_t stage_rows = compact_stage_rows(n_docs, ix.k);
    auto grid_of = [&](int64_t work) {
        int64_t g = (work + 255) / 256;
        return (unsigned)(g > (int64_t)sm_count * 8 ? (int64_t)sm_count * 8 : (g < 1 ? 1 : g));
    };
    DSK_LAUNCH(compact_count_kernel, grid_of(n_words), 256, 0, s, removed, n_words, n_docs, word_cnt);
    cudaError_t e = launch_exclusive_scan(word_cnt, n_words, word_ptr, scratch, s);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(compact_remap_kernel, grid_of(n_docs), 256, 0, s, removed, n_docs, word_ptr, remap, new2old);
    e = cudaMemcpyAsync(m, word_ptr + n_words, sizeof(int64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess || *m == n_docs) return e;   // nothing was removed: rows and tables stay as they are
    // Move the rows in place, a chunk of new numbers [a, b) at a time: gather the chunk's source rows into the staging area,
    // then write them to rows [a, b).  Safe because new numbers keep the old order: the source row s of new number t has
    // s >= t >= a, the earlier chunks wrote only rows < a, and every later chunk's sources are rows >= b.
    for (int64_t a = 0; a < *m; a += stage_rows) {
        const int64_t b = a + stage_rows < *m ? a + stage_rows : *m;
        DSK_LAUNCH(compact_gather_kernel, grid_of((b - a) * 32), 256, 0, s, ix.sig, ix.k, new2old, a, b, stage);
        e = cudaMemcpyAsync(ix.sig + a * ix.k, stage, (size_t)(b - a) * ix.k * 4, cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return e;
    }
    // empty tables (as dsk_lsh_create leaves them), then rows 0..m-1 re-inserted from the index's own storage
    e = cudaMemsetAsync(ix.slots, 0xFF, (size_t)ix.b * ix.cap_slots * 2 * sizeof(uint64_t), s);
    if (e == cudaSuccess) e = launch_lsh_insert(ix, ix.sig, 0, *m, sm_count, s);
    return e;
}

}  // namespace dsk

// ---- insert_unique: the streaming dedup loop over a batch --------------------------------------------------------------
// for each row j of the batch, in order: keep j (insert it) iff no remaining document of the index and no row j' < j of the
// batch that was kept is a candidate of j with eq >= min_count.  Three relations decide it:
//   stage A       the self-join's QUERY_BEST walk of every row against the index (removal-aware): a row with a kept
//                 candidate there is DROPPED whatever the batch holds, and its (idx, eq) is the index's side of its match;
//   batch pairs   a second LshDev over the batch rows themselves (a table in the caller's workspace, filled by
//                 lsh_insert_kernel, which skips its row copy because the rows already are the table's rows), whose
//                 PAIRS_COUNT / PAIRS_FILL walk lists every row's earlier partners d < j with eq >= min_count as CSR;
//   resolution    statuses UNDECIDED -> KEPT / DROPPED: a row with a KEPT earlier partner is DROPPED, a row whose earlier
//                 partners are all DROPPED (or that has none) is KEPT, any other row waits.
// A status is written once, from UNDECIDED to final, and a decision is taken from final statuses only, so by induction in
// row order every decision is the loop's, whichever order the threads visit the rows in and whichever of the other threads'
// writes of the same round they see: statuses are read and written with relaxed atomics.  The smallest undecided row can
// always decide, so every round decides at least one row; a drift chain (row j's only partner is j - 1) of length L takes
// about L rounds.  The rounds run as kUniqueSweeps grid-wide sweeps (one launch each, no host synchronisation), the last
// of which lists the rows still undecided; one CTA then loops over that list, round after round, separated by
// __syncthreads, until it is empty.  No CTA ever waits for another.  The statuses and both schedules (unique_sweep,
// unique_resolve) are dsk_common.cuh's, shared with MinHashLSHBloom's insert_unique.
namespace dsk {

// Decides row j from the statuses of its earlier partners pidx[ptr[j] .. ptr[j + 1]); false: j stays undecided.
__device__ __forceinline__ bool unique_decide(const int64_t *ptr, const int32_t *pidx, int32_t *st, int64_t j) {
    bool open = false;
    for (int64_t p = ptr[j]; p < ptr[j + 1]; ++p) {
        const int32_t s = ld_relaxed(st + pidx[p]);
        if (s == kKept) {
            st_relaxed(st + j, kDropped);
            return true;
        }
        open = open || s == kUndecided;
    }
    if (open) return false;
    st_relaxed(st + j, kKept);
    return true;
}

// st[j] = DROPPED for a row with a kept candidate in the index (stage A), else UNDECIDED
__global__ void __launch_bounds__(256) unique_init_kernel(const int32_t *__restrict__ aidx, int64_t n, int32_t *st) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
        st[j] = aidx[j] >= 0 ? kDropped : kUndecided;
}

// one grid-wide round over every undecided row; list != nullptr: appends the rows that stay undecided (in any order)
__global__ void __launch_bounds__(256) unique_sweep_kernel(const int64_t *__restrict__ ptr, const int32_t *__restrict__ pidx,
                                                           int32_t *st, int64_t n, int32_t *list, unsigned *list_n) {
    unique_sweep([&](int64_t j) { return unique_decide(ptr, pidx, st, j); }, st, n, list, list_n);
}

__global__ void __launch_bounds__(kResolveThreads) unique_resolve_kernel(const int64_t *__restrict__ ptr,
                                                                         const int32_t *__restrict__ pidx, int32_t *st,
                                                                         int32_t *list, int32_t *spare,
                                                                         const unsigned *list_n) {
    unique_resolve([&](int64_t j) { return unique_decide(ptr, pidx, st, j); }, list, spare, list_n);
}

// flags[j] = 1 for a kept row (the exclusive scan of the flags numbers the kept rows), kept[j] the caller's copy
__global__ void __launch_bounds__(256) unique_flags_kernel(const int32_t *__restrict__ st, int64_t n,
                                                           int64_t *__restrict__ flags, uint8_t *__restrict__ kept) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        const bool k = st[j] == kKept;
        flags[j] = k;
        kept[j] = k;
    }
}

// A kept row: match / eq = -1, new2old[rank] = j.  A dropped row: the best of stage A's (idx, eq) and its KEPT earlier
// partners (n0 + rank, eq) -- the largest eq, then the smallest document number, so an indexed document (< n0) wins a tie.
__global__ void __launch_bounds__(256) unique_match_kernel(const int32_t *__restrict__ st, const int64_t *__restrict__ ptr,
                                                           const int32_t *__restrict__ pidx, const int32_t *__restrict__ peq,
                                                           const int32_t *__restrict__ aidx, const int32_t *__restrict__ aeq,
                                                           const int64_t *__restrict__ rank, int64_t n0, int64_t n,
                                                           int32_t *__restrict__ match, int32_t *__restrict__ eq,
                                                           int32_t *__restrict__ new2old) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        if (st[j] == kKept) {
            match[j] = -1;
            eq[j] = -1;
            new2old[rank[j]] = (int32_t)j;
            continue;
        }
        int32_t bd = aidx[j], be = aeq[j];
        for (int64_t p = ptr[j]; p < ptr[j + 1]; ++p) {
            const int32_t d = pidx[p];
            if (st[d] != kKept) continue;
            const int32_t c = (int32_t)(n0 + rank[d]), e = peq[p];
            if (e > be || (e == be && c < bd)) { bd = c; be = e; }
        }
        match[j] = bd;
        eq[j] = be;
    }
}

// workspace of a batch of n rows: the batch table's slots [b][cap_slots][2] u64 and next [n][b] i32 | stage A's idx, eq
// i32[n] | statuses i32[n] | kept flags i64[n] | ranks i64[n + 1] | scan scratch i64[n / 1024 + 2] | two lists i32[n] |
// new -> old i32[n] | the list counter.  Each part 256-byte aligned.
static int64_t unique_cap_slots(int64_t n) {
    int64_t c = 2;
    while (c < 2 * n) c <<= 1;
    return c;
}

struct UniqueWs {
    LshDev bt;   // the batch table (sig = the batch rows)
    int32_t *aidx, *aeq, *st, *list, *spare, *new2old;
    int64_t *flags, *rank, *scratch;
    unsigned *list_n;
};

static UniqueWs unique_ws(void *ws, const LshDev &ix, const uint32_t *sig, int64_t n, size_t *bytes) {
    UniqueWs w{};
    char *p = static_cast<char *>(ws);
    size_t off = 0;
    auto take = [&](size_t sz) { char *q = p ? p + off : nullptr; off += align256(sz); return q; };
    w.bt.cap_slots = unique_cap_slots(n);
    w.bt.slots = reinterpret_cast<uint64_t *>(take((size_t)ix.b * w.bt.cap_slots * 16));
    w.bt.next = reinterpret_cast<int32_t *>(take((size_t)n * ix.b * 4));
    w.bt.sig = const_cast<uint32_t *>(sig);   // read only: lsh_insert_kernel does not copy rows onto themselves
    w.bt.cap_docs = n;
    w.bt.k = ix.k;
    w.bt.b = ix.b;
    w.bt.r = ix.r;
    w.aidx = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.aeq = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.st = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.flags = reinterpret_cast<int64_t *>(take((size_t)n * 8));
    w.rank = reinterpret_cast<int64_t *>(take((size_t)(n + 1) * 8));
    w.scratch = reinterpret_cast<int64_t *>(take((size_t)(n / 1024 + 2) * 8));
    w.list = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.spare = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.new2old = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.list_n = reinterpret_cast<unsigned *>(take(16));
    if (bytes) *bytes = off;
    return w;
}

size_t lsh_unique_workspace_bytes(const LshDev &ix, int64_t n) {
    if (n <= 0) return 0;
    size_t bytes = 0;
    unique_ws(nullptr, ix, nullptr, n, &bytes);
    return bytes;
}

static unsigned unique_grid(int64_t work, int sm_count) {
    int64_t g = (work + 255) / 256;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    return (unsigned)(g < 1 ? 1 : g);
}

// Builds the batch table over sig (n rows), runs stage A against the first n_docs documents of ix, and writes counts[j] =
// the number of row j's earlier partners in the batch.  No synchronisation.
cudaError_t lsh_unique_count(const LshDev &ix, int sw, int64_t n_docs, const uint32_t *sig, int64_t n, int min_count,
                             void *ws, int64_t *counts, const uint32_t *removed, int sm_count, cudaStream_t s) {
    const UniqueWs w = unique_ws(ws, ix, sig, n, nullptr);
    cudaError_t e = cudaMemsetAsync(w.bt.slots, 0xFF, (size_t)ix.b * w.bt.cap_slots * 16, s);   // empty key, head -1
    if (e == cudaSuccess) e = launch_lsh_insert(w.bt, sig, 0, n, sm_count, s);
    if (e == cudaSuccess)
        e = launch_lsh_query_pairs(ix, sw, sig, n, n_docs, min_count, nullptr, nullptr, w.aidx, w.aeq, removed, sm_count, s);
    if (e == cudaSuccess) e = launch_lsh_pairs(w.bt, sw, n, min_count, counts, nullptr, nullptr, nullptr, nullptr, sm_count, s);
    return e;
}

// After lsh_unique_count and the scan of its counts into ptr: fills the batch pairs (pidx / peq), resolves the statuses,
// writes kept / match / eq and new -> old, and returns *m = the number of kept rows.  Synchronises s once, to read m.
cudaError_t lsh_unique_resolve(const LshDev &ix, int sw, int64_t n_docs, const uint32_t *sig, int64_t n, int min_count, void *ws,
                               const int64_t *ptr, int32_t *pidx, int32_t *peq, uint8_t *kept, int32_t *match, int32_t *eq,
                               int64_t *m, int sm_count, cudaStream_t s) {
    const UniqueWs w = unique_ws(ws, ix, sig, n, nullptr);
    const unsigned grid = unique_grid(n, sm_count);
    cudaError_t e = launch_lsh_pairs(w.bt, sw, n, min_count, nullptr, ptr, pidx, peq, nullptr, sm_count, s);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(unique_init_kernel, grid, 256, 0, s, w.aidx, n, w.st);
    e = cudaMemsetAsync(w.list_n, 0, sizeof(unsigned), s);
    if (e != cudaSuccess) return e;
    for (int round = 0; round < kUniqueSweeps; ++round) {
        const bool last = round == kUniqueSweeps - 1;
        DSK_LAUNCH(unique_sweep_kernel, grid, 256, 0, s, ptr, (const int32_t *)pidx, w.st, n, last ? w.list : nullptr,
                   w.list_n);
    }
    DSK_LAUNCH(unique_resolve_kernel, 1, kResolveThreads, 0, s, ptr, (const int32_t *)pidx, w.st, w.list, w.spare,
               (const unsigned *)w.list_n);
    DSK_LAUNCH(unique_flags_kernel, grid, 256, 0, s, (const int32_t *)w.st, n, w.flags, kept);
    e = launch_exclusive_scan(w.flags, n, w.rank, w.scratch, s);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(unique_match_kernel, grid, 256, 0, s, (const int32_t *)w.st, ptr, (const int32_t *)pidx,
               (const int32_t *)peq, (const int32_t *)w.aidx, (const int32_t *)w.aeq, (const int64_t *)w.rank, n_docs, n,
               match, eq, w.new2old);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(m, w.rank + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return e;
}

// After lsh_unique_resolve: the m kept rows gathered into the index's storage behind its n_docs documents, then inserted
// there as documents n_docs .. n_docs + m - 1 (lsh_insert_kernel's copy is a self-copy).  The caller checked the capacity.
cudaError_t lsh_unique_insert(const LshDev &ix, int64_t n_docs, const uint32_t *sig, int64_t n, int64_t m, void *ws,
                              int sm_count, cudaStream_t s) {
    if (m <= 0) return cudaSuccess;
    const UniqueWs w = unique_ws(ws, ix, sig, n, nullptr);
    uint32_t *dst = ix.sig + n_docs * ix.k;
    DSK_LAUNCH(compact_gather_kernel, unique_grid(m * 32, sm_count), 256, 0, s, sig, ix.k, (const int32_t *)w.new2old,
               (int64_t)0, m, dst);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = launch_lsh_insert(ix, dst, n_docs, m, sm_count, s);
    return e;
}

}  // namespace dsk

// ---- MinHashLSHEnsemble: containment search over size partitions (lshensemble.py:189-249) ---------------------------------
// The reference keeps num_part x |rs| MinHashLSH indexes: indexes[p][r] holds the sets of size partition p, banded as
// (num_perm // r, r), and query(m, size) unions, over every partition p with an upper bound, the first b bands of
// indexes[p][r] with (b, r) = params[searchsorted(xqs, upper_p / size)].  Here the N sets are numbered in size-sorted order,
// so partition p is the range [part_start[p], part_start[p + 1]) of set numbers, and their rows are held once.  For each
// distinct r there is one set of b_r = num_perm // r band tables over all N sets, keyed by (partition, band, r-tuple): the
// fingerprint of ensemble_fp is band_fp's with the partition in the seed's high word, so a chain holds the members of one
// reference bucket indexes[p][r].hashtables[band][H] (plus fingerprint collisions, which the tuple check and the partition
// range drop).  map[d] translates set number d back to the caller's row.
namespace dsk {

__device__ __forceinline__ uint64_t ensemble_fp(const uint32_t *v, int r, int band, int part) {
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (uint64_t)band ^ ((uint64_t)(uint32_t)part << 32);
    for (int q = 0; q < r; ++q) h = (h ^ v[q]) * 0xFF51AFD7ED558CCDull + 0x2545F4914F6CDD1Dull;
    h = lsh_mix64(h);
    return h == kEmptyKey ? h - 1 : h;
}

// the partition of set number d: the last p with part_start[p] <= d (empty partitions have part_start[p] == part_start[p+1])
__device__ __forceinline__ int ensemble_part(const int64_t *part_start, int num_part, int64_t d) {
    int lo = 0, hi = num_part;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(part_start + mid) <= d) lo = mid;
        else hi = mid;
    }
    return lo;
}

// thread <-> (set d, band): the claim and chain update of lsh_insert_kernel, with the partition-keyed fingerprint.  The rows
// are in the table's storage already (gathered in size order), so they are only read.
__global__ void __launch_bounds__(256) ensemble_insert_kernel(const LshDev ix, const int64_t *__restrict__ part_start,
                                                              int num_part, int64_t n) {
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    const int64_t n_pairs = n * ix.b;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pairs; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t d = p / ix.b;
        const int band = (int)(p - d * ix.b);
        const int part = ensemble_part(part_start, num_part, d);
        const uint64_t fp = ensemble_fp(ix.sig + d * ix.k + band * ix.r, ix.r, band, part);
        uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
        uint64_t slot = lsh_mix64(fp) & mask;
        while (true) {
            const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long *>(tab + 2 * slot),
                                                      (unsigned long long)kEmptyKey, (unsigned long long)fp);
            if (prev == kEmptyKey || prev == fp) break;
            slot = (slot + 1) & mask;
        }
        const int32_t old = atomicExch(reinterpret_cast<int32_t *>(tab + 2 * slot + 1), (int32_t)d);
        ix.next[d * ix.b + band] = old;
    }
}

enum { ENS_COUNT = 0, ENS_FILL = 1, ENS_FILL_EQ = 2 };

// warp <-> item (query q, partition p) = q * num_part + p, lane <-> band < b (bands beyond 32 in further rounds), the query
// row staged in shared memory.  sel[item] is the row of the (b, r) table for the pair (-1, or any value outside the table:
// the partition is not queried).  Each lane probes its band's table of the chosen r with the partition-keyed fingerprint
// and walks the chain to its next candidate d: inside p's range, the tuple really equal, and no earlier band j < band with
// equal tuples (the first matching band among the first b emits it, the set union of MinHashLSH._query_b).  Then, as in
// lsh_pairs_kernel, the warp writes the pending candidates of all lanes together (ENS_FILL_EQ first counts eq for each of
// them over the two K-word rows).
//   ENS_COUNT    counts[item] = number of candidates
//   ENS_FILL     out_idx[ptr[item] ...) = map[d], in no particular order
//   ENS_FILL_EQ  the same, and out_eq at the same positions = number of the K positions where the rows agree
template <int MODE>
__global__ void __launch_bounds__(256) ensemble_query_kernel(const EnsembleDev en, const uint32_t *__restrict__ qsig,
                                                             int64_t nq, const int32_t *__restrict__ sel,
                                                             int64_t *__restrict__ counts, const int64_t *__restrict__ ptr,
                                                             int32_t *__restrict__ out_idx, int32_t *__restrict__ out_eq) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_rows, 16);   // [warps][k]
    const int lane = threadIdx.x & 31;
    const int k = en.tab[0].k;
    uint32_t *row = s_rows + (int64_t)(threadIdx.x >> 5) * k;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const unsigned below = (1u << lane) - 1u;
    const int64_t n_items = nq * en.num_part;
    for (int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < n_items; item += warps) {
        const int64_t q = item / en.num_part;
        const int part = (int)(item - q * en.num_part);
        const int s = sel[item];
        const int64_t lo = en.part_start[part], hi = en.part_start[part + 1];
        if (s < 0 || s >= en.n_params || lo >= hi) {   // warp-uniform
            if (MODE == ENS_COUNT && lane == 0) counts[item] = 0;
            continue;
        }
        const int nb = en.pb[s];
        const LshDev &ix = en.tab[en.pt[s]];
        const uint64_t mask = (uint64_t)ix.cap_slots - 1;
        const uint32_t *qrow = qsig + q * k;
        __syncwarp();
        for (int w = lane; w < k; w += 32) row[w] = qrow[w];
        __syncwarp();
        int64_t total = 0;   // candidates so far (the same in every lane)
        for (int band0 = 0; band0 < nb; band0 += 32) {
            const int band = band0 + lane;
            const uint32_t *qt = row + band * ix.r;
            int32_t d = -1;
            if (band < nb) {
                const uint64_t fp = ensemble_fp(qt, ix.r, band, part);
                const uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
                uint64_t slot = lsh_mix64(fp) & mask;
                while (true) {
                    const uint64_t kk = tab[2 * slot];
                    if (kk == fp) { d = *reinterpret_cast<const int32_t *>(tab + 2 * slot + 1); break; }
                    if (kk == kEmptyKey) break;
                    slot = (slot + 1) & mask;
                }
            }
            while (true) {
                int32_t cand = -1;
                while (d >= 0) {
                    const int32_t cur = d;
                    d = ix.next[(int64_t)cur * ix.b + band];
                    if (cur >= lo && cur < hi) {
                        const uint32_t *drow = ix.sig + (int64_t)cur * k;
                        if (tuple_eq(drow + band * ix.r, qt, ix.r)) {
                            bool dup = false;
                            for (int j = 0; j < band && !dup; ++j)
                                dup = tuple_eq(drow + j * ix.r, row + j * ix.r, ix.r);
                            if (!dup) { cand = cur; break; }
                        }
                    }
                }
                const unsigned pending = __ballot_sync(0xFFFFFFFFu, cand >= 0);
                if (pending == 0u) break;
                int eq = 0;
                if (MODE == ENS_FILL_EQ) {
                    for (unsigned m = pending; m; m &= m - 1u) {
                        const int src = __ffs(m) - 1;
                        const uint32_t *crow = ix.sig + (int64_t)__shfl_sync(0xFFFFFFFFu, cand, src) * k;
                        int e = 0;
                        for (int w = lane; w < k; w += 32) e += crow[w] == row[w];
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xFFFFFFFFu, e, o);
                        if (lane == src) eq = e;
                    }
                }
                if (MODE != ENS_COUNT && cand >= 0) {
                    const int64_t pos = ptr[item] + total + __popc(pending & below);
                    out_idx[pos] = en.map[cand];
                    if (MODE == ENS_FILL_EQ) out_eq[pos] = eq;
                }
                total += __popc(pending);
            }
        }
        if (MODE == ENS_COUNT && lane == 0) counts[item] = total;
    }
}

// Gathers the n rows into size order (sig[t] = rows[order[t]]), copies order as the map, and fills every table set.
cudaError_t ensemble_index(const EnsembleDev &en, const uint32_t *rows, const int32_t *order, int64_t n, int sm_count,
                           cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const LshDev &t0 = en.tab[0];
    auto grid_of = [&](int64_t work) {
        int64_t g = (work + 255) / 256;
        return (unsigned)(g > (int64_t)sm_count * 8 ? (int64_t)sm_count * 8 : (g < 1 ? 1 : g));
    };
    DSK_LAUNCH(compact_gather_kernel, grid_of(n * 32), 256, 0, s, rows, t0.k, order, (int64_t)0, n, t0.sig);
    cudaError_t e = cudaMemcpyAsync(en.map, order, (size_t)n * 4, cudaMemcpyDeviceToDevice, s);
    for (int t = 0; t < en.n_tabs && e == cudaSuccess; ++t) {
        const LshDev &ix = en.tab[t];
        e = cudaMemsetAsync(ix.slots, 0xFF, (size_t)ix.b * ix.cap_slots * 16, s);   // empty key, head -1
        if (e != cudaSuccess) break;
        DSK_LAUNCH(ensemble_insert_kernel, grid_of(n * ix.b), 256, 0, s, ix, (const int64_t *)en.part_start, en.num_part, n);
        e = cudaGetLastError();
    }
    return e;
}

// counts != nullptr: counts[item] for the nq * num_part items; else the fill of idx (and eq, if not null) at ptr[item].
cudaError_t ensemble_query(const EnsembleDev &en, const uint32_t *qsig, int64_t nq, const int32_t *sel, int64_t *counts,
                           const int64_t *ptr, int32_t *idx, int32_t *eq, int sm_count, cudaStream_t s) {
    const int64_t n_items = nq * en.num_part;
    if (n_items <= 0) return cudaSuccess;
    const int k = en.tab[0].k;
    int w = 8;
    while (w > 1 && (size_t)w * k * 4 > 48 * 1024) w >>= 1;
    const size_t smem = (size_t)w * k * 4;
    int64_t g = (n_items + w - 1) / w;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    const unsigned grid = (unsigned)g;
    cudaError_t e;
    if (counts) {
        e = cudaFuncSetAttribute(ensemble_query_kernel<ENS_COUNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH(ensemble_query_kernel<ENS_COUNT>, grid, 32 * w, smem, s, en, qsig, nq, sel, counts, nullptr, nullptr,
                   nullptr);
    } else if (eq) {
        e = cudaFuncSetAttribute(ensemble_query_kernel<ENS_FILL_EQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH(ensemble_query_kernel<ENS_FILL_EQ>, grid, 32 * w, smem, s, en, qsig, nq, sel, nullptr, ptr, idx, eq);
    } else {
        e = cudaFuncSetAttribute(ensemble_query_kernel<ENS_FILL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH(ensemble_query_kernel<ENS_FILL>, grid, 32 * w, smem, s, en, qsig, nq, sel, nullptr, ptr, idx, nullptr);
    }
    return cudaGetLastError();
}

// ---- containment estimates of the ensemble's candidates ---------------------------------------------------------------------
// c = j * (s_q + s_x) / (s_q * (1 + j)), j = eq / K: the inverse of the map t -> t / (1 + x/q - t) that turns a containment
// into the Jaccard value the (b, r) table was chosen for (lshensemble.py's _false_positive_probability), so c estimates
// |Q & X| / |Q|.  Evaluated as the Python expression over ints and floats is: every operation rounded on its own (no FMA
// contraction, no reciprocal), the int sum s_q + s_x exact (both sizes below 2^62) and converted once.
__device__ __forceinline__ double containment_est(int eq, int k, int64_t sq, int64_t sx) {
    const double j = __ddiv_rn((double)eq, (double)k);
    return __ddiv_rn(__dmul_rn(j, __ll2double_rn(sq + sx)), __dmul_rn(__ll2double_rn(sq), __dadd_rn(1.0, j)));
}

// ensemble_query_kernel's walk of one (query, partition) item with table row s, the query row in row[0..k): lane <-> band < b
// (further rounds beyond 32), the chain walk to each lane's next candidate (inside [lo, hi), not set number `skip`, the tuple
// really equal, no earlier band equal), and emit(pending, cand) for each round of candidates, warp-uniformly.
template <class Emit>
__device__ __forceinline__ void ensemble_walk(const EnsembleDev &en, const uint32_t *row, int part, int s, int64_t lo,
                                              int64_t hi, int64_t skip, int lane, Emit &&emit) {
    const int k = en.tab[0].k;
    const int nb = en.pb[s];
    const LshDev &ix = en.tab[en.pt[s]];
    const uint64_t mask = (uint64_t)ix.cap_slots - 1;
    for (int band0 = 0; band0 < nb; band0 += 32) {
        const int band = band0 + lane;
        const uint32_t *qt = row + band * ix.r;
        int32_t d = -1;
        if (band < nb) {
            const uint64_t fp = ensemble_fp(qt, ix.r, band, part);
            const uint64_t *tab = ix.slots + (int64_t)band * ix.cap_slots * 2;
            uint64_t slot = lsh_mix64(fp) & mask;
            while (true) {
                const uint64_t kk = tab[2 * slot];
                if (kk == fp) { d = *reinterpret_cast<const int32_t *>(tab + 2 * slot + 1); break; }
                if (kk == kEmptyKey) break;
                slot = (slot + 1) & mask;
            }
        }
        while (true) {
            int32_t cand = -1;
            while (d >= 0) {
                const int32_t cur = d;
                d = ix.next[(int64_t)cur * ix.b + band];
                if (cur >= lo && cur < hi && cur != skip) {
                    const uint32_t *drow = ix.sig + (int64_t)cur * k;
                    if (tuple_eq(drow + band * ix.r, qt, ix.r)) {
                        bool dup = false;
                        for (int j = 0; j < band && !dup; ++j)
                            dup = tuple_eq(drow + j * ix.r, row + j * ix.r, ix.r);
                        if (!dup) { cand = cur; break; }
                    }
                }
            }
            const unsigned pending = __ballot_sync(0xFFFFFFFFu, cand >= 0);
            if (pending == 0u) break;
            emit(pending, cand);
        }
    }
}

// eq of each pending lane's candidate against row[0..k), the warp comparing one candidate's row at a time (ENS_FILL_EQ's)
__device__ __forceinline__ int ensemble_pending_eq(const uint32_t *sig, int k, const uint32_t *row, unsigned pending,
                                                   int32_t cand, int lane) {
    int eq = 0;
    for (unsigned m = pending; m; m &= m - 1u) {
        const int src = __ffs(m) - 1;
        const uint32_t *crow = sig + (int64_t)__shfl_sync(0xFFFFFFFFu, cand, src) * k;
        int e = 0;
        for (int w = lane; w < k; w += 32) e += crow[w] == row[w];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xFFFFFFFFu, e, o);
        if (lane == src) eq = e;
    }
    return eq;
}

enum { ENSC_COUNT = 0, ENSC_FILL = 1 };

// warp <-> item, as ensemble_query_kernel, keeping the candidates x with containment_est(eq, K, s_q, s_x) >= min_c; s_x =
// set_sizes[map[x]] (the caller's row order).  SELF = false: item q * num_part + p of the nq query rows, s_q = qsizes[q].
// SELF = true: the walk goes over set numbers t (nq = n): the query is the index's own row t, s_q = set_sizes[map[t]], set t
// itself is skipped (by number: an identical row is still a candidate) and the item is written (and sel read) at
// map[t] * num_part + p, so the output is in the caller's row order.
//   ENSC_COUNT  counts[item] = number of kept candidates (eq is only counted when min_c > 0: every c is >= 0)
//   ENSC_FILL   out_idx / out_eq / out_c [ptr[item] ...) = row, eq and c of each kept candidate, in no particular order
template <int MODE, bool SELF>
__global__ void __launch_bounds__(256) ensemble_containment_kernel(
        const EnsembleDev en, const uint32_t *__restrict__ qsig, int64_t nq, const int64_t *__restrict__ qsizes,
        const int32_t *__restrict__ sel, const int64_t *__restrict__ set_sizes, double min_c, int64_t *__restrict__ counts,
        const int64_t *__restrict__ ptr, int32_t *__restrict__ out_idx, int32_t *__restrict__ out_eq,
        double *__restrict__ out_c) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_rows, 16);   // [warps][k]
    const int lane = threadIdx.x & 31;
    const int k = en.tab[0].k;
    uint32_t *row = s_rows + (int64_t)(threadIdx.x >> 5) * k;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const unsigned below = (1u << lane) - 1u;
    const int64_t n_items = nq * en.num_part;
    const bool need_eq = MODE == ENSC_FILL || min_c > 0.0;
    for (int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < n_items; item += warps) {
        const int64_t q = item / en.num_part;
        const int part = (int)(item - q * en.num_part);
        const int64_t out_item = SELF ? (int64_t)en.map[q] * en.num_part + part : item;
        const int s = sel[out_item];
        const int64_t lo = en.part_start[part], hi = en.part_start[part + 1];
        if (s < 0 || s >= en.n_params || lo >= hi) {   // warp-uniform
            if (MODE == ENSC_COUNT && lane == 0) counts[out_item] = 0;
            continue;
        }
        const uint32_t *qrow = SELF ? en.tab[0].sig + q * k : qsig + q * k;
        const int64_t sq = SELF ? set_sizes[en.map[q]] : qsizes[q];
        __syncwarp();
        for (int w = lane; w < k; w += 32) row[w] = qrow[w];
        __syncwarp();
        int64_t total = 0;   // kept candidates so far (the same in every lane)
        ensemble_walk(en, row, part, s, lo, hi, SELF ? q : -1, lane, [&](unsigned pending, int32_t cand) {
            int eq = 0;
            int32_t x = -1;
            double c = 0.0;
            if (need_eq) {
                eq = ensemble_pending_eq(en.tab[0].sig, k, row, pending, cand, lane);
                if (cand >= 0) {
                    x = en.map[cand];
                    c = containment_est(eq, k, sq, set_sizes[x]);
                }
            }
            const bool keep = cand >= 0 && (!need_eq || c >= min_c);
            const unsigned kept = __ballot_sync(0xFFFFFFFFu, keep);
            if (MODE == ENSC_FILL && keep) {
                const int64_t pos = ptr[out_item] + total + __popc(kept & below);
                out_idx[pos] = x;
                out_eq[pos] = eq;
                out_c[pos] = c;
            }
            total += __popc(kept);
        });
        if (MODE == ENSC_COUNT && lane == 0) counts[out_item] = total;
    }
}

// The warp-held list of ensemble_containment_topk_kernel: lane j holds entry j as (best_c, best_x, best_eq), -1.0 / -1 / -1
// while empty, in the order larger c, then smaller row x; topk_insert's shift, keyed by (c, x).
__device__ __forceinline__ void topk_insert_c(double &best_c, int32_t &best_x, int32_t &best_eq, double c, int32_t x, int eq,
                                              int lane, int topk) {
    const bool better = lane < topk && (best_c > c || (best_c == c && best_x < x));
    const int at = __popc(__ballot_sync(0xFFFFFFFFu, better));   // entries before (c, x)
    if (at < topk) {
        const double uc = __shfl_up_sync(0xFFFFFFFFu, best_c, 1);
        const int32_t ux = __shfl_up_sync(0xFFFFFFFFu, best_x, 1);
        const int32_t ue = __shfl_up_sync(0xFFFFFFFFu, best_eq, 1);
        if (lane == at) { best_c = c; best_x = x; best_eq = eq; }
        else if (lane > at) { best_c = uc; best_x = ux; best_eq = ue; }
    }
}

// warp <-> query q: the walk of each of its partitions in turn, every candidate with c >= min_c into the warp-held list (a
// query's candidates are disjoint across partitions, and the first-band rule emits each once within one, so no merge is
// needed); lanes < topk store out_idx / out_eq / out_c [q * topk + lane].  An index never built (map == nullptr) pads.
__global__ void __launch_bounds__(256) ensemble_containment_topk_kernel(
        const EnsembleDev en, const uint32_t *__restrict__ qsig, int64_t nq, const int64_t *__restrict__ qsizes,
        const int32_t *__restrict__ sel, const int64_t *__restrict__ set_sizes, double min_c, int topk,
        int32_t *__restrict__ out_idx, int32_t *__restrict__ out_eq, double *__restrict__ out_c) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_rows, 16);   // [warps][k]
    const int lane = threadIdx.x & 31;
    const int k = en.tab[0].k;
    uint32_t *row = s_rows + (int64_t)(threadIdx.x >> 5) * k;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int n_part = en.map ? en.num_part : 0;
    for (int64_t q = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); q < nq; q += warps) {
        const int64_t sq = qsizes[q];
        __syncwarp();
        for (int w = lane; w < k; w += 32) row[w] = qsig[q * k + w];
        __syncwarp();
        double best_c = -1.0;
        int32_t best_x = -1, best_eq = -1;
        for (int part = 0; part < n_part; ++part) {
            const int s = sel[q * en.num_part + part];
            const int64_t lo = en.part_start[part], hi = en.part_start[part + 1];
            if (s < 0 || s >= en.n_params || lo >= hi) continue;   // warp-uniform
            ensemble_walk(en, row, part, s, lo, hi, -1, lane, [&](unsigned pending, int32_t cand) {
                const int eq = ensemble_pending_eq(en.tab[0].sig, k, row, pending, cand, lane);
                const int32_t x = cand >= 0 ? en.map[cand] : -1;
                const double c = x >= 0 ? containment_est(eq, k, sq, set_sizes[x]) : -1.0;
                for (unsigned m = __ballot_sync(0xFFFFFFFFu, x >= 0 && c >= min_c); m; m &= m - 1u) {
                    const int src = __ffs(m) - 1;
                    topk_insert_c(best_c, best_x, best_eq, __shfl_sync(0xFFFFFFFFu, c, src),
                                  __shfl_sync(0xFFFFFFFFu, x, src), __shfl_sync(0xFFFFFFFFu, eq, src), lane, topk);
                }
            });
        }
        if (lane < topk) {
            out_idx[q * topk + lane] = best_x;
            out_eq[q * topk + lane] = best_eq;
            out_c[q * topk + lane] = best_c;
        }
    }
}

// counts != nullptr: counts[item] for the nq * num_part items; else the fill of idx / eq / c at ptr[item].  qsig == nullptr:
// the self-join (nq = the number of sets, the index's own rows and set_sizes as the queries' sizes).
cudaError_t ensemble_containment(const EnsembleDev &en, const uint32_t *qsig, int64_t nq, const int64_t *qsizes,
                                 const int32_t *sel, const int64_t *set_sizes, double min_c, int64_t *counts,
                                 const int64_t *ptr, int32_t *idx, int32_t *eq, double *c, int sm_count, cudaStream_t s) {
    const int64_t n_items = nq * en.num_part;
    if (n_items <= 0) return cudaSuccess;
    const int k = en.tab[0].k;
    int w = 8;
    while (w > 1 && (size_t)w * k * 4 > 48 * 1024) w >>= 1;
    const size_t smem = (size_t)w * k * 4;
    int64_t g = (n_items + w - 1) / w;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    const unsigned grid = (unsigned)g;
    auto launch = [&](auto kernel) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH(kernel, grid, 32 * w, smem, s, en, qsig, nq, qsizes, sel, set_sizes, min_c, counts, ptr, idx, eq, c);
        return cudaGetLastError();
    };
    if (qsig) return counts ? launch(ensemble_containment_kernel<ENSC_COUNT, false>)
                            : launch(ensemble_containment_kernel<ENSC_FILL, false>);
    return counts ? launch(ensemble_containment_kernel<ENSC_COUNT, true>) : launch(ensemble_containment_kernel<ENSC_FILL, true>);
}

cudaError_t ensemble_containment_topk(const EnsembleDev &en, const uint32_t *qsig, int64_t nq, const int64_t *qsizes,
                                      const int32_t *sel, const int64_t *set_sizes, double min_c, int topk, int32_t *idx,
                                      int32_t *eq, double *c, int sm_count, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    const int k = en.tab[0].k;
    int w = 8;
    while (w > 1 && (size_t)w * k * 4 > 48 * 1024) w >>= 1;
    const size_t smem = (size_t)w * k * 4;
    int64_t g = (nq + w - 1) / w;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    cudaError_t e = cudaFuncSetAttribute(ensemble_containment_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(ensemble_containment_topk_kernel, (unsigned)g, 32 * w, smem, s, en, qsig, nq, qsizes, sel, set_sizes, min_c,
               topk, idx, eq, c);
    return cudaGetLastError();
}

}  // namespace dsk

// ---- MinHashLSHEnsemble's size partitioner (lshensemble.py:81-120 = lshensemble_partition.py:54-196) ----------------------
// Over the D distinct set sizes (ascending) with their counts: cost[l, u] = sum over i in [l, u] of
// (sizes[u] - sizes[i]) / sizes[u] * counts[i], as numpy evaluates it (each operation rounded on its own, the sum numpy's
// float64 pairwise sum), stored as a column-major upper triangle (entry (l, u) at u(u+1)/2 + l); then the reference's dynamic
// programme over p = 2 .. num_part-1 intervals and its back-tracking, every argmin taking the first index among equal values.
// The triangle is D^3/6 additions and D^2/2 divisions; the programme and the back-tracking read it num_part times.
namespace dsk {

// numpy's pairwise_sum of a[0..n) for n <= 128 (a leaf): below 8 elements a sequential sum from 0.0; else eight accumulators
// seeded with a[0..8) and stepping by 8, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n mod 8 tail in order
__device__ __forceinline__ double np_leaf_sum(const double *a, int n) {
    if (n < 8) {
        double res = 0.0;
        for (int i = 0; i < n; ++i) res = __dadd_rn(res, a[i]);
        return res;
    }
    double r0 = a[0], r1 = a[1], r2 = a[2], r3 = a[3], r4 = a[4], r5 = a[5], r6 = a[6], r7 = a[7];
    const int m = n - n % 8;
    for (int i = 8; i < m; i += 8) {
        r0 = __dadd_rn(r0, a[i]);
        r1 = __dadd_rn(r1, a[i + 1]);
        r2 = __dadd_rn(r2, a[i + 2]);
        r3 = __dadd_rn(r3, a[i + 3]);
        r4 = __dadd_rn(r4, a[i + 4]);
        r5 = __dadd_rn(r5, a[i + 5]);
        r6 = __dadd_rn(r6, a[i + 6]);
        r7 = __dadd_rn(r7, a[i + 7]);
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r0, r1), __dadd_rn(r2, r3)), __dadd_rn(__dadd_rn(r4, r5), __dadd_rn(r6, r7)));
    for (int i = m; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
}

// numpy's pairwise_sum of a[0..n): above 128 elements, the sum of the first n2 = n/2 - (n/2) % 8 plus the sum of the rest.
// The recursion runs on an explicit stack, left half first, so the leaves are met in ascending order: pos is where the next
// one starts, rest[d] the length of level d's right half while its left half is summed (-1 once it is summed into left[d]).
constexpr int kPairwiseDepth = 48;   // each level at least halves n - 8: enough for any n < 2^48
__device__ __forceinline__ double np_pairwise_sum(const double *a, int64_t n) {
    int64_t rest[kPairwiseDepth];
    double left[kPairwiseDepth];
    int depth = 0;
    int64_t pos = 0;
    while (true) {
        while (n > 128) {
            int64_t n2 = n / 2;
            n2 -= n2 % 8;
            rest[depth++] = n - n2;
            n = n2;
        }
        double v = np_leaf_sum(a + pos, (int)n);
        pos += n;
        while (depth > 0 && rest[depth - 1] < 0) v = __dadd_rn(left[--depth], v);
        if (depth == 0) return v;
        left[depth - 1] = v;
        n = rest[depth - 1];
        rest[depth - 1] = -1;
    }
}

constexpr int kPartitionCostThreads = 512;
constexpr int64_t kPartitionSmemTerms = 28 * 1024;    // a column's terms fit the shared memory of one CTA up to D = 28672
constexpr int64_t kPartitionTermRows = 512;           // beyond that: CTAs of the cost launch, one global row of D terms each

// CTA <-> column u (largest first, grid-stride): the u + 1 terms of the column, term i = (sizes[u] - sizes[i]) / sizes[u] *
// counts[i] (every operation rounded on its own: no contraction into an FMA, no reciprocal), into shared memory (or the CTA's
// row of g_terms), then thread <-> entry l: cost[l, u] = the pairwise sum of terms l..u.  row0[u] = cost[0, u] (if not null).
template <bool SMEM_TERMS>
__global__ void __launch_bounds__(kPartitionCostThreads) partition_cost_kernel(const int64_t *__restrict__ sizes,
                                                                               const int64_t *__restrict__ counts, int64_t n,
                                                                               double *__restrict__ cost,
                                                                               double *__restrict__ row0, double *g_terms) {
    DSK_DYNAMIC_SMEM_T(double, s_terms, 16);
    double *t = SMEM_TERMS ? s_terms : g_terms + (int64_t)blockIdx.x * n;
    for (int64_t u = n - 1 - blockIdx.x; u >= 0; u -= gridDim.x) {
        const double top = __ll2double_rn(sizes[u]);
        __syncthreads();   // the previous column's sums are done with t
        for (int64_t i = threadIdx.x; i <= u; i += blockDim.x)
            t[i] = __dmul_rn(__ddiv_rn(__dsub_rn(top, __ll2double_rn(sizes[i])), top), __ll2double_rn(counts[i]));
        __syncthreads();
        double *col = cost + u * (u + 1) / 2;
        for (int64_t l = threadIdx.x; l <= u; l += blockDim.x) {
            const double v = np_pairwise_sum(t + l, u - l + 1);
            col[l] = v;
            if (l == 0 && row0) row0[u] = v;
        }
    }
}

// warp <-> u in [p-1, n): tab[u] = min over u1 in [p-2, u-1] of prev[u1] + cost[u1 + 1, u] (column u is contiguous).  Entries
// u < p-1 are not written (the caller zeroes them, as the reference's zero-initialised matrix).
__global__ void __launch_bounds__(256) partition_dp_kernel(const double *__restrict__ cost, const double *__restrict__ prev,
                                                           double *__restrict__ tab, int p, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = n - 1 - ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)); u >= p - 1; u -= warps) {
        const double *col = cost + u * (u + 1) / 2 + 1;   // col[u1] = cost[u1 + 1, u]
        double best = (double)INFINITY;
        for (int64_t u1 = p - 2 + lane; u1 < u; u1 += 32) {
            const double v = __dadd_rn(prev[u1], col[u1]);
            best = v < best ? v : best;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double w = __shfl_xor_sync(0xFFFFFFFFu, best, o);
            best = w < best ? w : best;
        }
        if (lane == 0) tab[u] = best;
    }
}

// (v, i) pairs: the smaller value, the smaller index among equal values
__device__ __forceinline__ void argmin_first(double &v, int64_t &i, double w, int64_t j) {
    if (w < v || (w == v && j < i)) { v = w; i = j; }
}

// one CTA: the reference's back-tracking.  u = n-1; for p = num_part .. 2: u1 = the first argmin over [p-2, u-1] of
// prev[u1] + cost[u1 + 1, u], the upper index of partition p-2, then u = u1.  prev is the (p-1)-interval table for the
// first step and, as in the reference (lshensemble_partition.py:158-166), the p-interval table after it, where the
// recurrence used p-1; its entries below p-1 are the zeros.  tab row q (q = 1 .. num_part-1) is the q-interval table at
// tab + (q-1) * n, row 1 = cost[0, .].
__global__ void __launch_bounds__(256) partition_backtrack_kernel(const double *__restrict__ cost,
                                                                  const double *__restrict__ tab, int num_part, int64_t n,
                                                                  int64_t *__restrict__ upper) {
    __shared__ double s_v[8];
    __shared__ int64_t s_i[8];
    __shared__ int64_t s_u;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t u = n - 1;
    if (threadIdx.x == 0) upper[num_part - 1] = u;
    for (int p = num_part; p >= 2; --p) {
        const double *prev = tab + (int64_t)((p == num_part ? p - 1 : p) - 1) * n;
        const double *col = cost + u * (u + 1) / 2 + 1;
        double bv = (double)INFINITY;
        int64_t bi = INT64_MAX;
        for (int64_t u1 = p - 2 + threadIdx.x; u1 < u; u1 += blockDim.x) {
            const double v = __dadd_rn(prev[u1], col[u1]);
            if (v < bv) { bv = v; bi = u1; }   // ascending in each thread: the strict test keeps the first
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            argmin_first(bv, bi, __shfl_xor_sync(0xFFFFFFFFu, bv, o), __shfl_xor_sync(0xFFFFFFFFu, bi, o));
        if (lane == 0) { s_v[warp] = bv; s_i[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            const int nw = (int)(blockDim.x >> 5);
            bv = lane < nw ? s_v[lane] : (double)INFINITY;
            bi = lane < nw ? s_i[lane] : INT64_MAX;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
                argmin_first(bv, bi, __shfl_xor_sync(0xFFFFFFFFu, bv, o), __shfl_xor_sync(0xFFFFFFFFu, bi, o));
            if (lane == 0) { upper[p - 2] = bi; s_u = bi; }
        }
        __syncthreads();
        u = s_u;
    }
}

bool partition_terms_in_smem(int64_t n) { return n <= kPartitionSmemTerms; }
int64_t partition_term_rows(int64_t n) { return partition_terms_in_smem(n) ? 0 : (n < kPartitionTermRows ? n : kPartitionTermRows); }

// The triangle into cost; with tab != nullptr (2 <= num_part < n) also the tables (num_part - 1 rows of n) and the upper
// index of each partition into upper[num_part].  g_terms: partition_term_rows(n) rows of n doubles (or nullptr if 0).
cudaError_t ensemble_partition(const int64_t *sizes, const int64_t *counts, int64_t n, int num_part, double *cost, double *tab,
                               double *g_terms, int64_t *upper, int sm_count, cudaStream_t s) {
    cudaError_t e;
    if (partition_terms_in_smem(n)) {
        const int smem = (int)(n * 8);
        e = cudaFuncSetAttribute(partition_cost_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH(partition_cost_kernel<true>, (unsigned)n, kPartitionCostThreads, (size_t)smem, s, sizes, counts, n, cost,
                   tab, nullptr);
    } else {
        DSK_LAUNCH(partition_cost_kernel<false>, (unsigned)partition_term_rows(n), kPartitionCostThreads, 0, s, sizes, counts,
                   n, cost, tab, g_terms);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess || !tab) return e;
    if (num_part > 2) e = cudaMemsetAsync(tab + n, 0, (size_t)(num_part - 2) * n * 8, s);
    int64_t g = (n + 7) / 8;
    if (g > (int64_t)sm_count * 16) g = (int64_t)sm_count * 16;
    for (int p = 2; p < num_part && e == cudaSuccess; ++p) {
        DSK_LAUNCH(partition_dp_kernel, (unsigned)g, 256, 0, s, (const double *)cost, (const double *)(tab + (int64_t)(p - 2) * n),
                   tab + (int64_t)(p - 1) * n, p, n);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(partition_backtrack_kernel, 1, 256, 0, s, (const double *)cost, (const double *)tab, num_part, n, upper);
    return cudaGetLastError();
}

}  // namespace dsk
