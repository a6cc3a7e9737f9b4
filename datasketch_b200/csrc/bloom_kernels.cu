// bloom_kernels.cu -- MinHashLSHBloom on the device (SURVEY.md section 8 f3).
//
// The reference keys each band's Bloom filter with  x = sum(hashvalues[start:end]) % (2^61 - 1)
// (datasketch/lsh_bloom.py:94-106 insert, :108-118 query; `_mersenne_prime` :20).  `band_sums_kernel` is that
// codec over a whole signature matrix (HBM-bound: 4K bytes in, 8b bytes out per document); the fused
// `bloom_bands_kernel` goes on to set / test the k probe bits of every band's table, so the [n, b] key matrix
// never reaches memory.  The bit tables are this library's own (the reference delegates them to pybloomfilter,
// whose file format is not reproduced): classic k-probe Bloom filters, one per band, double hashing.
#include <algorithm>

#include "dsk_common.cuh"

namespace dsk {

constexpr uint64_t kBloomP61 = (1ull << 61) - 1;

__device__ __forceinline__ uint64_t mod_p61(uint64_t x) {   // x % (2^61 - 1) for any 64-bit x
    uint64_t s = (x & kBloomP61) + (x >> 61);
    return s >= kBloomP61 ? s - kBloomP61 : s;
}

__device__ __forceinline__ uint64_t bloom_mix(uint64_t h) {
    h ^= h >> 33; h *= 0xFF51AFD7ED558CCDull; h ^= h >> 33; h *= 0xC4CEB9FE1A85EC53ull; h ^= h >> 33;
    return h;
}

// warp <-> document: the b*r values the bands use are read once with coalesced loads into the warp's slice of shared
// memory (STAGED), then lane j sums band j.  A row too long for shared memory is summed straight from global memory.
// x < 2^32 * r, so the uint64 sum cannot wrap for r <= 2^32 and `% p` is the conditional fold below.
template <int MODE, bool STAGED>   // MODE 0 = write the keys, 1 = insert into the tables, 2 = query the tables
__global__ void __launch_bounds__(256) bloom_bands_kernel(const uint32_t *__restrict__ sig, int64_t n, int k, int b, int r,
                                                          uint64_t *__restrict__ keys, uint32_t *__restrict__ bits,
                                                          uint64_t words_per_table, uint64_t n_bits, int n_hashes,
                                                          uint8_t *__restrict__ hit) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_row, 16);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int br = b * r;
    uint32_t *row = s_row + (size_t)w * br;
    for (int64_t i = (int64_t)blockIdx.x * nw + w; i < n; i += (int64_t)gridDim.x * nw) {
        const uint32_t *g = sig + i * k;
        if (STAGED) {
            __syncwarp();
            for (int c = lane; c < br; c += 32) row[c] = __ldg(g + c);
            __syncwarp();
        }
        bool any = false;
        for (int j = lane; j < b; j += 32) {
            uint64_t x = 0;
            if (STAGED) {
                const uint32_t *v = row + j * r;
                for (int q = 0; q < r; ++q) x += v[q];
            } else {
                const uint32_t *v = g + (int64_t)j * r;
                for (int q = 0; q < r; ++q) x += __ldg(v + q);
            }
            x = mod_p61(x);
            if (MODE == 0) {
                keys[i * b + j] = x;
            } else {
                const uint64_t h1 = bloom_mix(x ^ 0x9E3779B97F4A7C15ull), h2 = bloom_mix(x + 0xD6E8FEB86659FD93ull) | 1ull;
                uint32_t *tab = bits + (uint64_t)j * words_per_table;
                bool all = true;
                for (int q = 0; q < n_hashes; ++q) {
                    const uint64_t pos = (h1 + (uint64_t)q * h2) % n_bits;
                    const uint32_t m = 1u << (pos & 31);
                    if (MODE == 1) atomicOr(tab + (pos >> 5), m);
                    else all = all && (tab[pos >> 5] & m) != 0;
                }
                any = any || all;
            }
        }
        if (MODE == 2) {   // a match in ANY band makes the document a duplicate candidate (lsh_bloom.py:365-371)
            any = __any_sync(0xFFFFFFFFu, any);
            if (lane == 0) hit[i] = any ? 1 : 0;
        }
    }
}

// keys only: thread <-> (document, band), the r values read straight from global memory (neighbouring threads read
// neighbouring bands of the same row, so the row's sectors are shared in L1) -- the layout band_fingerprint_kernel reaches
// 76-85 % of the HBM copy peak with; the warp-per-document kernel above leaves 32 - b lanes idle in the summing loop.
__global__ void __launch_bounds__(256) band_sums_kernel(const uint32_t *__restrict__ sig, int64_t n, int k, int b, int r,
                                                        uint64_t *__restrict__ keys) {
    const int64_t total = n * b, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t i = e / b;
        const int band = (int)(e - i * b);
        const uint32_t *v = sig + i * k + (int64_t)band * r;
        uint64_t x = 0;
        for (int q = 0; q < r; ++q) x += __ldg(v + q);
        keys[e] = mod_p61(x);
    }
}

template <int MODE>
static cudaError_t launch_bloom_mode(int warps, size_t smem, const uint32_t *sig, int64_t n, int k, int b, int r,
                                     uint64_t *keys, uint32_t *bits, uint64_t words_per_table, uint64_t n_bits,
                                     int n_hashes, uint8_t *hit, int grid, cudaStream_t s) {
    if (smem == 0) {
        DSK_LAUNCH((bloom_bands_kernel<MODE, false>), grid, warps * 32, 0, s, sig, n, k, b, r, keys, bits, words_per_table, n_bits, n_hashes, hit);
        return cudaGetLastError();
    }
    const cudaError_t e = cudaFuncSetAttribute(bloom_bands_kernel<MODE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH((bloom_bands_kernel<MODE, true>), grid, warps * 32, smem, s, sig, n, k, b, r, keys, bits, words_per_table, n_bits, n_hashes, hit);
    return cudaGetLastError();
}

// Each warp stages the b*r values it sums (not the whole num_perm-long row): 8 warps per CTA while their slices fit in
// 96 KB, fewer for longer rows.  A row longer than 96 KB (b*r > 24576) is read from global memory instead, as
// band_sums_kernel does, so any b*r <= num_perm launches.  smem = 0: the rows are not staged.
static void bloom_warps(int b, int r, int *warps, size_t *smem) {
    constexpr size_t kStageBytes = 96 * 1024;
    const size_t row_bytes = (size_t)b * r * 4;
    *warps = 8;
    while (*warps > 1 && *warps * row_bytes > kStageBytes) *warps >>= 1;
    *smem = *warps * row_bytes;
    if (*smem > kStageBytes) {
        *warps = 8;
        *smem = 0;
    }
}

static cudaError_t launch_bloom_bands(int mode, const uint32_t *sig, int64_t n, int k, int b, int r, uint64_t *keys,
                                      uint32_t *bits, uint64_t words_per_table, uint64_t n_bits, int n_hashes,
                                      uint8_t *hit, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    int warps;
    size_t smem;
    bloom_warps(b, r, &warps, &smem);
    const int grid = (int)std::min<int64_t>((n + warps - 1) / warps, (int64_t)sm_count * 8);
    if (mode == 0) return launch_bloom_mode<0>(warps, smem, sig, n, k, b, r, keys, bits, words_per_table, n_bits, n_hashes, hit, grid, s);
    if (mode == 1) return launch_bloom_mode<1>(warps, smem, sig, n, k, b, r, keys, bits, words_per_table, n_bits, n_hashes, hit, grid, s);
    return launch_bloom_mode<2>(warps, smem, sig, n, k, b, r, keys, bits, words_per_table, n_bits, n_hashes, hit, grid, s);
}

cudaError_t launch_band_sums(const uint32_t *sig, int64_t n, int k, int b, int r, uint64_t *keys, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int64_t total = n * b;
    const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count * 16);
    DSK_LAUNCH(band_sums_kernel, grid, 256, 0, s, sig, n, k, b, r, keys);
    return cudaGetLastError();
}
cudaError_t launch_bloom_insert(const uint32_t *sig, int64_t n, int k, int b, int r, uint32_t *bits, uint64_t words_per_table,
                                uint64_t n_bits, int n_hashes, int sm_count, cudaStream_t s) {
    return launch_bloom_bands(1, sig, n, k, b, r, nullptr, bits, words_per_table, n_bits, n_hashes, nullptr, sm_count, s);
}
cudaError_t launch_bloom_query(const uint32_t *sig, int64_t n, int k, int b, int r, const uint32_t *bits,
                               uint64_t words_per_table, uint64_t n_bits, int n_hashes, uint8_t *hit, int sm_count,
                               cudaStream_t s) {
    return launch_bloom_bands(2, sig, n, k, b, r, nullptr, const_cast<uint32_t *>(bits), words_per_table, n_bits, n_hashes, hit,
                              sm_count, s);
}

// ---- insert_unique: the query-then-insert loop over a batch (DESIGN.md §4i) ------------------------------------------------
// for each row j of the batch, in order: if no band of j has all its probe bits set, insert j.  A probe bit of row j is set
// when the loop reaches j iff it was set before the call or some KEPT row j' < j probes the same (band, position).  Three
// stages, every buffer in the caller's workspace, no host synchronisation:
//   probe     warp <-> row, staged as bloom_bands_kernel: a row with a band whose bits are all set in the tables before the
//             call is DROPPED and emits nothing; any other row emits one entry (band, pos, row) per probe bit not set
//             there, chained per (band, pos) key through an open-addressing table (atomicCAS claim, atomicExch head);
//   resolve   statuses UNDECIDED -> KEPT / DROPPED with dsk_common.cuh's schedule: a row is DROPPED when some band has a
//             KEPT earlier setter for each of its missing bits; KEPT when every band has a missing bit whose earlier setters
//             are all DROPPED (or that has none); otherwise it waits.  The induction of §4e holds as it is: decisions use
//             final statuses only, and the smallest undecided row's earlier rows are all final;
//   commit    entry <-> thread: each entry of a KEPT row ORs its bit into its table (the pre-set bits need no write, so the
//             signatures are not read again), and keep[j] = (st[j] == KEPT).
// Entries are numbered e = (row * b + band) * n_hashes + q, so an entry's row and band follow from e; the key of (band, pos)
// is band * n_bits + pos (the C-ABI rejects geometries where b * n_bits does not fit 64 bits).
struct BloomUniqueWs {
    uint64_t *key;       // [cap] (band, pos) keys, kEmptyKey = free
    int32_t *head;       // [cap] the last entry chained to the key, -1 = none
    int32_t *slot;       // [n * b * n_hashes] entry -> its key's slot, -1 = the bit was set before the call
    int32_t *next;       // [n * b * n_hashes] the next entry of the same key, -1 = end
    int32_t *st, *list, *spare;   // [n] statuses, and the resolving CTA's two row lists
    unsigned *list_n;
    int64_t cap;         // 2 * n * b * n_hashes slots: load factor <= 1/2
};

// workspace of a batch of n rows, each part 256-byte aligned: keys u64[cap] | heads i32[cap] | entry slots i32[E] | entry
// links i32[E] | statuses, two lists i32[n] | the list counter, with E = n * b * n_hashes and cap = 2E:
// 24 * E + 8 * E + 12 * n bytes plus alignment.  The caller checked E <= kBloomUniqueMaxEntries.
static BloomUniqueWs bloom_unique_ws(void *ws, int64_t n, int b, int n_hashes, size_t *bytes) {
    BloomUniqueWs w{};
    char *p = static_cast<char *>(ws);
    size_t off = 0;
    auto take = [&](size_t sz) { char *q = p ? p + off : nullptr; off += (sz + 255) & ~(size_t)255; return q; };
    const int64_t entries = n * b * n_hashes;
    w.cap = 2 * entries;
    w.key = reinterpret_cast<uint64_t *>(take((size_t)w.cap * 8));
    w.head = reinterpret_cast<int32_t *>(take((size_t)w.cap * 4));
    w.slot = reinterpret_cast<int32_t *>(take((size_t)entries * 4));
    w.next = reinterpret_cast<int32_t *>(take((size_t)entries * 4));
    w.st = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.list = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.spare = reinterpret_cast<int32_t *>(take((size_t)n * 4));
    w.list_n = reinterpret_cast<unsigned *>(take(16));
    if (bytes) *bytes = off;
    return w;
}

size_t bloom_unique_workspace_bytes(int64_t n, int b, int n_hashes) {
    if (n <= 0) return 0;
    size_t bytes = 0;
    bloom_unique_ws(nullptr, n, b, n_hashes, &bytes);
    return bytes;
}

template <bool STAGED>
__device__ __forceinline__ uint64_t bloom_band_key(const uint32_t *row, const uint32_t *g, int j, int r) {
    uint64_t x = 0;
    if (STAGED) {
        const uint32_t *v = row + j * r;
        for (int q = 0; q < r; ++q) x += v[q];
    } else {
        const uint32_t *v = g + (int64_t)j * r;
        for (int q = 0; q < r; ++q) x += __ldg(v + q);
    }
    return mod_p61(x);
}

template <bool STAGED>
__global__ void __launch_bounds__(256) bloom_unique_probe_kernel(const uint32_t *__restrict__ sig, int64_t n, int k, int b,
                                                                 int r, const uint32_t *__restrict__ bits,
                                                                 uint64_t words_per_table, uint64_t n_bits, int n_hashes,
                                                                 const BloomUniqueWs w) {
    DSK_DYNAMIC_SMEM_T(uint32_t, s_row, 16);
    const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int br = b * r;
    uint32_t *row = s_row + (size_t)wi * br;
    for (int64_t i = (int64_t)blockIdx.x * nw + wi; i < n; i += (int64_t)gridDim.x * nw) {
        const uint32_t *g = sig + i * k;
        if (STAGED) {
            __syncwarp();
            for (int c = lane; c < br; c += 32) row[c] = __ldg(g + c);
            __syncwarp();
        }
        bool covered = false;   // some band has every probe bit set before the call: the loop drops the row
        for (int j = lane; j < b; j += 32) {
            const uint64_t x = bloom_band_key<STAGED>(row, g, j, r);
            const uint64_t h1 = bloom_mix(x ^ 0x9E3779B97F4A7C15ull), h2 = bloom_mix(x + 0xD6E8FEB86659FD93ull) | 1ull;
            const uint32_t *tab = bits + (uint64_t)j * words_per_table;
            bool all = true;
            for (int q = 0; q < n_hashes && all; ++q) {
                const uint64_t pos = (h1 + (uint64_t)q * h2) % n_bits;
                all = (tab[pos >> 5] >> (pos & 31)) & 1u;
            }
            covered = covered || all;
        }
        covered = __any_sync(0xFFFFFFFFu, covered);
        if (lane == 0) w.st[i] = covered ? kDropped : kUndecided;
        if (covered) continue;
        for (int j = lane; j < b; j += 32) {
            const uint64_t x = bloom_band_key<STAGED>(row, g, j, r);
            const uint64_t h1 = bloom_mix(x ^ 0x9E3779B97F4A7C15ull), h2 = bloom_mix(x + 0xD6E8FEB86659FD93ull) | 1ull;
            const uint32_t *tab = bits + (uint64_t)j * words_per_table;
            const int32_t e0 = (int32_t)((i * b + j) * n_hashes);
            for (int q = 0; q < n_hashes; ++q) {
                const uint64_t pos = (h1 + (uint64_t)q * h2) % n_bits;
                if ((tab[pos >> 5] >> (pos & 31)) & 1u) {
                    w.slot[e0 + q] = -1;
                    continue;
                }
                const uint64_t key = (uint64_t)j * n_bits + pos;
                uint64_t s = __umul64hi(lsh_mix64(key), (uint64_t)w.cap);
                while (true) {
                    const unsigned long long prev = atomicCAS((unsigned long long *)(w.key + s), kEmptyKey, key);
                    if (prev == kEmptyKey || prev == key) break;
                    if (++s == (uint64_t)w.cap) s = 0;
                }
                w.slot[e0 + q] = (int32_t)s;
                w.next[e0 + q] = atomicExch(w.head + s, e0 + q);
            }
        }
    }
}

// Decides row j (not dropped by the probe, so all its entries exist) from the final statuses of its bits' earlier setters.
__device__ __forceinline__ bool bloom_unique_decide(const BloomUniqueWs &w, int b, int n_hashes, int32_t *st, int64_t j) {
    const int per_row = b * n_hashes;
    const int32_t *es = w.slot + j * per_row;
    bool open = false;   // some band is neither covered nor free yet
    for (int t = 0; t < b; ++t) {
        bool covered = true, free = false;
        for (int q = 0; q < n_hashes; ++q) {
            const int32_t s = es[t * n_hashes + q];
            if (s < 0) continue;   // set before the call
            bool set = false, wait = false;
            for (int32_t e = w.head[s]; e >= 0; e = w.next[e]) {
                const int32_t d = e / per_row;
                if (d >= j) continue;   // only rows before j have set their bits when the loop reaches j
                const int32_t sd = ld_relaxed(st + d);
                if (sd == kKept) {
                    set = true;
                    break;
                }
                wait = wait || sd == kUndecided;
            }
            if (set) continue;
            covered = false;
            if (!wait) {   // no earlier row can set this bit: the band stays uncovered
                free = true;
                break;
            }
        }
        if (covered) {
            st_relaxed(st + j, kDropped);
            return true;
        }
        open = open || !free;
    }
    if (open) return false;
    st_relaxed(st + j, kKept);
    return true;
}

__global__ void __launch_bounds__(256) bloom_unique_sweep_kernel(const BloomUniqueWs w, int b, int n_hashes, int64_t n,
                                                                 int32_t *list) {
    int32_t *st = w.st;
    unique_sweep([&](int64_t j) { return bloom_unique_decide(w, b, n_hashes, st, j); }, st, n, list, w.list_n);
}

__global__ void __launch_bounds__(kResolveThreads) bloom_unique_resolve_kernel(const BloomUniqueWs w, int b, int n_hashes) {
    int32_t *st = w.st;
    unique_resolve([&](int64_t j) { return bloom_unique_decide(w, b, n_hashes, st, j); }, w.list, w.spare, w.list_n);
}

__global__ void __launch_bounds__(256) bloom_unique_commit_kernel(const BloomUniqueWs w, int64_t n, int b, int n_hashes,
                                                                  uint32_t *bits, uint64_t words_per_table, uint64_t n_bits,
                                                                  uint8_t *__restrict__ keep) {
    const int per_row = b * n_hashes;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, first = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t e = first; e < n * per_row; e += stride) {
        const int32_t i = (int32_t)e / per_row;
        if (w.st[i] != kKept) continue;
        const int32_t s = w.slot[e];
        if (s < 0) continue;
        const int t = ((int32_t)e - i * per_row) / n_hashes;
        const uint64_t pos = w.key[s] - (uint64_t)t * n_bits;
        atomicOr(bits + (uint64_t)t * words_per_table + (pos >> 5), 1u << (pos & 31));
    }
    for (int64_t j = first; j < n; j += stride) keep[j] = w.st[j] == kKept;
}

static unsigned bloom_unique_grid(int64_t work, int sm_count) {
    const int64_t g = std::min<int64_t>((work + 255) / 256, (int64_t)sm_count * 8);
    return (unsigned)std::max<int64_t>(g, 1);
}

cudaError_t bloom_unique(const uint32_t *sig, int64_t n, int k, int b, int r, uint32_t *bits, uint64_t words_per_table,
                         uint64_t n_bits, int n_hashes, void *ws, uint8_t *keep, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const BloomUniqueWs w = bloom_unique_ws(ws, n, b, n_hashes, nullptr);
    cudaError_t e = cudaMemsetAsync(w.key, 0xFF, (size_t)w.cap * 8, s);   // kEmptyKey
    if (e == cudaSuccess) e = cudaMemsetAsync(w.head, 0xFF, (size_t)w.cap * 4, s);   // -1
    if (e == cudaSuccess) e = cudaMemsetAsync(w.list_n, 0, sizeof(unsigned), s);
    if (e != cudaSuccess) return e;
    int warps;
    size_t smem;
    bloom_warps(b, r, &warps, &smem);
    const int pgrid = (int)std::min<int64_t>((n + warps - 1) / warps, (int64_t)sm_count * 8);
    if (smem == 0) {
        DSK_LAUNCH((bloom_unique_probe_kernel<false>), pgrid, warps * 32, 0, s, sig, n, k, b, r, bits, words_per_table, n_bits,
                   n_hashes, w);
    } else {
        e = cudaFuncSetAttribute(bloom_unique_probe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        DSK_LAUNCH((bloom_unique_probe_kernel<true>), pgrid, warps * 32, smem, s, sig, n, k, b, r, bits, words_per_table, n_bits,
                   n_hashes, w);
    }
    const unsigned grid = bloom_unique_grid(n, sm_count);
    for (int round = 0; round < kUniqueSweeps; ++round)
        DSK_LAUNCH(bloom_unique_sweep_kernel, grid, 256, 0, s, w, b, n_hashes, n, round == kUniqueSweeps - 1 ? w.list : nullptr);
    DSK_LAUNCH(bloom_unique_resolve_kernel, 1, kResolveThreads, 0, s, w, b, n_hashes);
    DSK_LAUNCH(bloom_unique_commit_kernel, bloom_unique_grid(n * b * n_hashes, sm_count), 256, 0, s, w, n, b, n_hashes, bits,
               words_per_table, n_bits, keep);
    return cudaGetLastError();
}

}  // namespace dsk
