// hash_core.cuh -- the token hashes as device functions over a byte reader, shared by the token kernels (sha1_kernels.cu,
// hash_kernels.cu) and the shingle kernels (shingle_kernels.cuh).
//
// A reader hands out the message bytes in order, one next() per byte; every core reads each byte exactly once, front to
// back, and is told the message length up front.  SpanReader reads a contiguous byte range; shingle_kernels.cuh has a reader
// that walks the words of a word n-gram and inserts the single spaces, so no shingle is ever copied to memory.
//   SHA-1              FIPS 180-4; sha1_hash32 / sha1_hash64 read the first 4 / 8 digest bytes little-endian
//   XXH32              xxHash specification (Y. Collet), 32-bit variant
//   MurmurHash3 x86_32 A. Appleby's public-domain MurmurHash3
#pragma once
#include "dsk_common.cuh"

namespace dsk {

struct SpanReader {
    const uint8_t *p;
    __device__ __forceinline__ uint32_t next() { return *p++; }
};

template <class R>
__device__ __forceinline__ uint32_t read_le32(R &rd) {
    const uint32_t b0 = rd.next(), b1 = rd.next(), b2 = rd.next(), b3 = rd.next();
    return b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
}

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

// byte p of the padded message (length len, total padded length plen); bytes below len come from the reader, in order
template <class R>
__device__ __forceinline__ uint32_t sha1_padded_byte(R &rd, int64_t len, int64_t plen, int64_t p) {
    if (p < len) return rd.next();
    if (p == len) return 0x80u;
    if (p >= plen - 8) {
        const uint64_t bits = (uint64_t)len * 8ull;
        return (uint32_t)((bits >> (8 * (plen - 1 - p))) & 0xFFu);
    }
    return 0u;
}

// the first two words of the SHA-1 digest of the len-byte message, as sha1_hash32 / sha1_hash64 read them (little-endian)
template <class R>
__device__ __forceinline__ void sha1_lo_hi(R &rd, int64_t len, uint32_t *lo, uint32_t *hi) {
    const int64_t plen = ((len + 8) / 64 + 1) * 64;
    uint32_t h0 = 0x67452301u, h1 = 0xEFCDAB89u, h2 = 0x98BADCFEu, h3 = 0x10325476u, h4 = 0xC3D2E1F0u;
    for (int64_t blk = 0; blk < plen; blk += 64) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int64_t p = blk + 4 * i;
            const uint32_t b0 = sha1_padded_byte(rd, len, plen, p), b1 = sha1_padded_byte(rd, len, plen, p + 1);
            const uint32_t b2 = sha1_padded_byte(rd, len, plen, p + 2), b3 = sha1_padded_byte(rd, len, plen, p + 3);
            w[i] = (b0 << 24) | (b1 << 16) | (b2 << 8) | b3;
        }
        uint32_t a = h0, b = h1, c = h2, e = h4, dd = h3;
#pragma unroll
        for (int i = 0; i < 80; ++i) {
            uint32_t wi;
            if (i < 16) wi = w[i];
            else {
                wi = rotl32(w[(i - 3) & 15] ^ w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15], 1);
                w[i & 15] = wi;
            }
            uint32_t f, k;
            if (i < 20) { f = (b & c) | (~b & dd); k = 0x5A827999u; }
            else if (i < 40) { f = b ^ c ^ dd; k = 0x6ED9EBA1u; }
            else if (i < 60) { f = (b & c) | (b & dd) | (c & dd); k = 0x8F1BBCDCu; }
            else { f = b ^ c ^ dd; k = 0xCA62C1D6u; }
            const uint32_t tmp = rotl32(a, 5) + f + e + k + wi;
            e = dd; dd = c; c = rotl32(b, 30); b = a; a = tmp;
        }
        h0 += a; h1 += b; h2 += c; h3 += dd; h4 += e;
    }
    // digest bytes are h0 (big endian), h1, ...; the reference reads the first 4 / 8 bytes little-endian
    *lo = __byte_perm(h0, 0, 0x0123);
    *hi = __byte_perm(h1, 0, 0x0123);
}

template <class R>
__device__ __forceinline__ uint32_t xxh32(R &rd, int64_t len, uint32_t seed) {
    constexpr uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
    int64_t i = 0;
    uint32_t h;
    if (len >= 16) {
        uint32_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
        for (; i + 16 <= len; i += 16) {
            v1 = rotl32(v1 + read_le32(rd) * P2, 13) * P1;
            v2 = rotl32(v2 + read_le32(rd) * P2, 13) * P1;
            v3 = rotl32(v3 + read_le32(rd) * P2, 13) * P1;
            v4 = rotl32(v4 + read_le32(rd) * P2, 13) * P1;
        }
        h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
    } else {
        h = seed + P5;
    }
    h += (uint32_t)len;
    for (; i + 4 <= len; i += 4) h = rotl32(h + read_le32(rd) * P3, 17) * P4;
    for (; i < len; ++i) h = rotl32(h + rd.next() * P5, 11) * P1;
    h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
    return h;
}

template <class R>
__device__ __forceinline__ uint32_t murmur3_32(R &rd, int64_t len, uint32_t seed) {
    constexpr uint32_t C1 = 0xcc9e2d51u, C2 = 0x1b873593u;
    uint32_t h = seed;
    int64_t i = 0;
    for (; i + 4 <= len; i += 4) {
        uint32_t k = read_le32(rd) * C1;
        k = rotl32(k, 15) * C2;
        h = rotl32(h ^ k, 13) * 5u + 0xe6546b64u;
    }
    const int tail = (int)(len - i);
    if (tail >= 1) {
        const uint32_t b0 = rd.next(), b1 = tail >= 2 ? rd.next() : 0u, b2 = tail == 3 ? rd.next() : 0u;
        uint32_t k = b0 | (b1 << 8) | (b2 << 16);
        k = rotl32(k * C1, 15) * C2;
        h ^= k;
    }
    h ^= (uint32_t)len;
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}

// the 32-bit token of one message under hash kind 0 (sha1_hash32), DSK_HASH_XXH32 or DSK_HASH_MURMUR3_32
template <int KIND, class R>
__device__ __forceinline__ uint32_t hash32(R &rd, int64_t len, uint32_t seed) {
    if (KIND == DSK_HASH_XXH32) return xxh32(rd, len, seed);
    if (KIND == DSK_HASH_MURMUR3_32) return murmur3_32(rd, len, seed);
    uint32_t lo, hi;
    sha1_lo_hi(rd, len, &lo, &hi);
    return lo;
}

}  // namespace dsk
