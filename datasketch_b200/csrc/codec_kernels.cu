// codec_kernels.cu -- HBM-bound signature codecs (sm_90a).
//
//  lean_pack / lean_unpack : [N,K] u32 signatures <-> LeanMinHash records `q i {K}I`
//                            (datasketch/lean_minhash.py:174-175, :201-214), any byte order.
//                            Tile kernel: 1-D TMA bulk load of a tile of rows into shared memory
//                            (cp.async.bulk + mbarrier), in-smem re-layout by all warps, 1-D TMA
//                            bulk store of the finished tile (cp.async.bulk.global.shared::cta).
//  band_keys_be            : [N,K] u32 -> [N, b, 8r] bytes: each band's r values as big-endian
//                            u64 (the dict keys MinHashLSH._H builds, lsh.py:344, :537-538).
//  band_fingerprints       : [N,K] u32 -> [N, b] u64 bucket key of each band's r-tuple (GPU bucketing;
//                            candidates are verified on the exact r-tuple, see lsh_kernels.cu).
#include <algorithm>

#include "dsk_common.cuh"

namespace dsk {

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// ---- LeanMinHash records --------------------------------------------------------------------
// One record = (K + 3) 32-bit words: seed lo, seed hi, K, then K hash values (little endian);
// for big-endian output every field is byte-reversed (the int64 seed also swaps its halves).
constexpr int kCodecThreads = 256;

struct LeanParams {
    const uint32_t *sig;   // [n, k]
    uint32_t *rec;         // [n, k + 3] words
    int64_t n;
    int k;
    int rows_per_tile;     // multiple of 4 (keeps every tile 16-byte aligned on both sides)
    uint32_t w0, w1, w2;   // header words, already in output byte order
    int big_endian;
    int64_t expect_seed;   // unpack: validated header (status flag on mismatch)
    int *status;           // unpack: set to 1 if any record header mismatches
};

constexpr int kLeanStages = 4;  // tiles in flight per CTA (loads) -- Little's law: ~100 KB in flight per SM

template <bool PACK>
__global__ void __launch_bounds__(kCodecThreads) lean_tile_kernel(const LeanParams p) {
    DSK_DYNAMIC_SMEM(smem);
    __shared__ __align__(8) uint64_t full[kLeanStages];
    const int K = p.k, RW = p.k + 3, R = p.rows_per_tile;
    const int in_rw = PACK ? K : RW, out_rw = PACK ? RW : K;
    const size_t in_words = (size_t)R * in_rw, out_words = (size_t)R * out_rw;
    // layout: in[S] | out[S]; every region starts 16-byte aligned (R % 4 == 0, K % 4 == 0 on this path)
    uint32_t *sin0 = reinterpret_cast<uint32_t *>(smem);
    uint32_t *sout0 = sin0 + kLeanStages * in_words;
    const uint32_t *gin = PACK ? p.sig : p.rec;
    uint32_t *gout = PACK ? p.rec : const_cast<uint32_t *>(p.sig);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = kCodecThreads / 32;
    const int64_t ntiles = (p.n + R - 1) / R;
    if (tid == 0) {
        for (int i = 0; i < kLeanStages; ++i) mbar_init(&full[i], 1);
        fence_mbar_init();
    }
    __syncthreads();

    auto load_tile = [&](int64_t t, int stage) {  // thread 0
        const int64_t r0 = t * R;
        const int nr = (int)min((int64_t)R, p.n - r0);
        const uint32_t bulk = (uint32_t)((size_t)nr * in_rw * 4) & ~15u;
        if (bulk) {
            mbar_arrive_expect_tx(&full[stage], bulk);
            bulk_g2s(sin0 + stage * in_words, gin + (size_t)r0 * in_rw, bulk, &full[stage]);
        } else {
            mbar_arrive(&full[stage]);
        }
    };

    if (tid == 0)
        for (int i = 0; i < kLeanStages; ++i) {
            const int64_t t = blockIdx.x + (int64_t)i * gridDim.x;
            if (t < ntiles) load_tile(t, i);
        }
    int64_t it = 0;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
        const int stage = (int)(it % kLeanStages);
        const uint32_t phase = (uint32_t)((it / kLeanStages) & 1);
        uint32_t *sin = sin0 + stage * in_words, *sout = sout0 + stage * out_words;
        const int64_t r0 = t * R;
        const int nr = (int)min((int64_t)R, p.n - r0);
        if (tid == 0) bulk_wait_read<kLeanStages - 1>();  // the store that last used sout[stage] has read it
        mbar_wait(&full[stage], phase);
        {   // bytes beyond the last 16-byte granule of a ragged final tile come by plain loads
            const uint32_t words = (uint32_t)((size_t)nr * in_rw), bulk_words = words & ~3u;
            if (tid < (int)(words - bulk_words)) sin[bulk_words + tid] = gin[(size_t)r0 * in_rw + bulk_words + tid];
        }
        __syncthreads();
        // re-layout: warp <-> record, lane <-> word (conflict-free on both sides)
        for (int r = warp; r < nr; r += nwarps) {
            const uint32_t *src = sin + (size_t)r * in_rw;
            uint32_t *dst = sout + (size_t)r * out_rw;
            if (PACK) {
                for (int c = lane; c < RW; c += 32) {
                    uint32_t v;
                    if (c >= 3) { v = src[c - 3]; if (p.big_endian) v = bswap32(v); }
                    else v = (c == 0) ? p.w0 : (c == 1) ? p.w1 : p.w2;
                    dst[c] = v;
                }
            } else {
                if (lane < 3) {
                    const uint32_t want = (lane == 0) ? p.w0 : (lane == 1) ? p.w1 : p.w2;
                    if (src[lane] != want) *p.status = 1;
                }
                for (int c = lane; c < K; c += 32) {
                    uint32_t v = src[c + 3];
                    if (p.big_endian) v = bswap32(v);
                    dst[c] = v;
                }
            }
        }
        fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA store
        __syncthreads();      // also: every reader of sin[stage] is done -> it can be refilled
        const uint32_t obytes = (uint32_t)((size_t)nr * out_rw * 4), obulk = obytes & ~15u;
        if (tid == 0) {
            if (obulk) bulk_s2g(gout + (size_t)r0 * out_rw, sout, obulk);
            bulk_commit();
            const int64_t tn = t + (int64_t)kLeanStages * gridDim.x;
            if (tn < ntiles) load_tile(tn, stage);
        }
        if (tid < (int)((obytes - obulk) / 4)) gout[(size_t)r0 * out_rw + obulk / 4 + tid] = sout[obulk / 4 + tid];
    }
    if (tid == 0) bulk_wait_read<0>();
}

// general fallback (any K, u32 or u64 input, any alignment): one thread per output word
__global__ void lean_pack_simple_kernel(const void *sig, int sig_is_u64, int64_t n, int k, uint32_t w0, uint32_t w1,
                                        uint32_t w2, int big_endian, uint32_t *rec) {
    const int rw = k + 3;
    const int64_t total = n * rw, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t r = e / rw;
        const int c = (int)(e - r * rw);
        uint32_t v;
        if (c >= 3) {
            v = sig_is_u64 ? (uint32_t) static_cast<const uint64_t *>(sig)[r * k + c - 3]
                           : static_cast<const uint32_t *>(sig)[r * k + c - 3];
            if (big_endian) v = bswap32(v);
        } else {
            v = (c == 0) ? w0 : (c == 1) ? w1 : w2;
        }
        rec[e] = v;
    }
}

__global__ void lean_unpack_simple_kernel(const uint32_t *rec, int64_t n, int k, uint32_t w0, uint32_t w1, uint32_t w2,
                                          int big_endian, void *sig, int sig_is_u64, int *status) {
    const int rw = k + 3;
    const int64_t total = n * rw, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t r = e / rw;
        const int c = (int)(e - r * rw);
        uint32_t v = rec[e];
        if (c >= 3) {
            if (big_endian) v = bswap32(v);
            if (sig_is_u64) static_cast<uint64_t *>(sig)[r * k + c - 3] = v;
            else static_cast<uint32_t *>(sig)[r * k + c - 3] = v;
        } else {
            const uint32_t want = (c == 0) ? w0 : (c == 1) ? w1 : w2;
            if (v != want) *status = 1;
        }
    }
}

// ---- LSH band keys --------------------------------------------------------------------------------
// warp <-> document, lane <-> value: coalesced 4-byte loads, coalesced 8-byte stores
__global__ void __launch_bounds__(256) band_keys_be_kernel(const uint32_t *__restrict__ sig, int64_t n, int k, int br,
                                                           uint2 *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
        const uint32_t *row = sig + i * k;
        uint2 *orow = out + i * br;
        for (int c0 = 0; c0 < br; c0 += 256) {  // 8 independent loads per lane before the first store
            uint32_t v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int c = c0 + u * 32 + lane;
                v[u] = c < br ? __ldg(row + c) : 0u;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int c = c0 + u * 32 + lane;
                if (c < br) orow[c] = make_uint2(0u, bswap32(v[u]));  // 00 00 00 00 b3 b2 b1 b0
            }
        }
    }
}

// The LSH index's bucket key of each band (band_fp, dsk_common.cuh: the tables' empty key remapped included); equal
// tuples <=> equal fingerprints up to 2^-64 collisions, which the LSH kernels resolve by comparing the tuples.
__global__ void __launch_bounds__(256) band_fingerprint_kernel(const uint32_t *__restrict__ sig, int64_t n, int k,
                                                               int b, int r, uint64_t *__restrict__ out) {
    const int64_t total = n * b, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t i = e / b;
        const int band = (int)(e - i * b);
        out[e] = band_fp(sig + i * k + (int64_t)band * r, r, band);
    }
}

// ---- b-bit MinHash blocks (datasketch/b_bit_minhash.py:78-92) ----------------------------------------
// block i of a row packs values [i*n, (i+1)*n) masked to b bits, value j at bit (n-1-j)*slot; n = 64/slot.
__global__ void __launch_bounds__(256) bbit_pack_kernel(const uint32_t *__restrict__ sig, int64_t n_rows, int k,
                                                        uint32_t bmask, int slot, int nblk,
                                                        uint64_t *__restrict__ out) {
    const int per = 64 / slot;
    const int64_t total = n_rows * nblk, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t row = e / nblk;
        const int blk = (int)(e - row * nblk);
        const uint32_t *v = sig + row * k + (int64_t)blk * per;
        const int cnt = min(per, k - blk * per);
        uint64_t w = 0;
        for (int j = 0; j < cnt; ++j) w |= (uint64_t)(v[j] & bmask) << ((per - 1 - j) * slot);
        out[e] = w;
    }
}

__global__ void __launch_bounds__(256) bbit_unpack_kernel(const uint64_t *__restrict__ blocks, int64_t n_rows, int k,
                                                          int slot, int nblk, uint32_t *__restrict__ sig) {
    const int per = 64 / slot;
    const uint64_t mask = slot == 64 ? ~0ull : ((1ull << slot) - 1);
    const int64_t total = n_rows * k, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int64_t row = e / k;
        const int c = (int)(e - row * k);
        const int blk = c / per, j = c - blk * per;
        sig[e] = (uint32_t)((blocks[row * nblk + blk] >> ((per - 1 - j) * slot)) & mask);
    }
}

cudaError_t launch_bbit_pack(const uint32_t *sig, int64_t n, int k, int b, int slot, uint64_t *out, int sm_count,
                             cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int per = 64 / slot, nblk = (k + per - 1) / per;
    const uint32_t bmask = b >= 32 ? 0xFFFFFFFFu : ((1u << b) - 1u);
    const int grid = (int)std::min<int64_t>((n * nblk + 255) / 256, (int64_t)sm_count * 16);
    DSK_LAUNCH(bbit_pack_kernel, grid, 256, 0, s, sig, n, k, bmask, slot, nblk, out);
    return cudaGetLastError();
}

cudaError_t launch_bbit_unpack(const uint64_t *blocks, int64_t n, int k, int slot, uint32_t *sig, int sm_count,
                               cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int per = 64 / slot, nblk = (k + per - 1) / per;
    const int grid = (int)std::min<int64_t>((n * k + 255) / 256, (int64_t)sm_count * 16);
    DSK_LAUNCH(bbit_unpack_kernel, grid, 256, 0, s, blocks, n, k, slot, nblk, sig);
    return cudaGetLastError();
}

// ---- launchers --------------------------------------------------------------------------------------
static void lean_header(int64_t seed, int k, int big_endian, uint32_t &w0, uint32_t &w1, uint32_t &w2) {
    const uint32_t lo = (uint32_t)(uint64_t)seed, hi = (uint32_t)((uint64_t)seed >> 32);
    if (big_endian) {
        w0 = __builtin_bswap32(hi); w1 = __builtin_bswap32(lo); w2 = __builtin_bswap32((uint32_t)k);
    } else {
        w0 = lo; w1 = hi; w2 = (uint32_t)k;
    }
}

static int lean_rows_per_tile(int k) {
    // kLeanStages x (in + out) tiles in ~68 KB so three CTAs share an SM
    const size_t per_row = (size_t)(2 * k + 3) * 4 * kLeanStages;
    int r = (int)((68 * 1024) / per_row) & ~3;
    if (r > 32) r = 32;
    return r;
}

cudaError_t launch_lean_pack(const void *sig, int sig_is_u64, int64_t n, int k, int64_t seed, int big_endian,
                             uint8_t *rec, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    uint32_t w0, w1, w2;
    lean_header(seed, k, big_endian, w0, w1, w2);
    const int R = lean_rows_per_tile(k);
    const bool tile_ok = !sig_is_u64 && (k % 4) == 0 && R >= 4 && ((uintptr_t)sig % 16) == 0 && ((uintptr_t)rec % 16) == 0;
    if (tile_ok) {
        LeanParams p{};
        p.sig = static_cast<const uint32_t *>(sig); p.rec = reinterpret_cast<uint32_t *>(rec);
        p.n = n; p.k = k; p.rows_per_tile = R; p.w0 = w0; p.w1 = w1; p.w2 = w2; p.big_endian = big_endian;
        const size_t smem = (size_t)R * (2 * k + 3) * 4 * kLeanStages;
        cudaError_t e = cudaFuncSetAttribute(lean_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        const int64_t ntiles = (n + R - 1) / R;
        const int grid = (int)std::min<int64_t>(ntiles, (int64_t)sm_count * 3);
        DSK_LAUNCH((lean_tile_kernel<true>), grid, kCodecThreads, smem, s, p);
    } else {
        const int64_t total = n * (k + 3);
        const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count * 16);
        DSK_LAUNCH(lean_pack_simple_kernel, grid, 256, 0, s, sig, sig_is_u64, n, k, w0, w1, w2, big_endian,
                                                     reinterpret_cast<uint32_t *>(rec));
    }
    return cudaGetLastError();
}

cudaError_t launch_lean_unpack(const uint8_t *rec, int64_t n, int k, int64_t seed, int big_endian, void *sig,
                               int sig_is_u64, int *d_status, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    uint32_t w0, w1, w2;
    lean_header(seed, k, big_endian, w0, w1, w2);
    const int R = lean_rows_per_tile(k);
    const bool tile_ok = !sig_is_u64 && (k % 4) == 0 && R >= 4 && ((uintptr_t)sig % 16) == 0 && ((uintptr_t)rec % 16) == 0;
    if (tile_ok) {
        LeanParams p{};
        p.sig = static_cast<const uint32_t *>(sig); p.rec = reinterpret_cast<uint32_t *>(const_cast<uint8_t *>(rec));
        p.n = n; p.k = k; p.rows_per_tile = R; p.w0 = w0; p.w1 = w1; p.w2 = w2; p.big_endian = big_endian;
        p.status = d_status;
        const size_t smem = (size_t)R * (2 * k + 3) * 4 * kLeanStages;
        cudaError_t e = cudaFuncSetAttribute(lean_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        const int64_t ntiles = (n + R - 1) / R;
        const int grid = (int)std::min<int64_t>(ntiles, (int64_t)sm_count * 3);
        DSK_LAUNCH((lean_tile_kernel<false>), grid, kCodecThreads, smem, s, p);
    } else {
        const int64_t total = n * (k + 3);
        const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count * 16);
        DSK_LAUNCH(lean_unpack_simple_kernel, grid, 256, 0, s, reinterpret_cast<const uint32_t *>(rec), n, k, w0, w1, w2,
                                                       big_endian, sig, sig_is_u64, d_status);
    }
    return cudaGetLastError();
}

cudaError_t launch_band_keys_be(const uint32_t *sig, int64_t n, int k, int b, int r, uint8_t *out, int sm_count,
                                cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int grid = (int)std::min<int64_t>((n + 7) / 8, (int64_t)sm_count * 8);
    DSK_LAUNCH(band_keys_be_kernel, grid, 256, 0, s, sig, n, k, b * r, reinterpret_cast<uint2 *>(out));
    return cudaGetLastError();
}

cudaError_t launch_band_fingerprints(const uint32_t *sig, int64_t n, int k, int b, int r, uint64_t *out, int sm_count,
                                     cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int64_t total = n * b;
    const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count * 16);
    DSK_LAUNCH(band_fingerprint_kernel, grid, 256, 0, s, sig, n, k, b, r, out);
    return cudaGetLastError();
}

}  // namespace dsk
