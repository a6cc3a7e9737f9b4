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
// band_sums_kernel does, so any b*r <= num_perm launches.
static cudaError_t launch_bloom_bands(int mode, const uint32_t *sig, int64_t n, int k, int b, int r, uint64_t *keys,
                                      uint32_t *bits, uint64_t words_per_table, uint64_t n_bits, int n_hashes,
                                      uint8_t *hit, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    constexpr size_t kStageBytes = 96 * 1024;
    const size_t row_bytes = (size_t)b * r * 4;
    int warps = 8;
    while (warps > 1 && warps * row_bytes > kStageBytes) warps >>= 1;
    size_t smem = warps * row_bytes;
    if (smem > kStageBytes) {
        warps = 8;
        smem = 0;
    }
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

}  // namespace dsk
