// shingle_kernels.cuh -- raw UTF-8 text to word or character n-gram tokens on the device (DESIGN.md §4m).
// Compiled once, as part of dsk_api.cu (the C-ABI that is its only caller); include it nowhere else.
//
// The definition is datasketch_b200/shingle.py:shingles(): words are str.split() (maximal runs of code points outside
// Python's 29 whitespace code points), a word n-gram is its words joined by one U+0020, a character n-gram is n code
// points, a document with 1 <= m < n units gives one shingle of all of them and an empty one gives none.  Each shingle
// becomes one 32-bit token, the token hash of its UTF-8 bytes, ready for the signature kernel.
//
// Every pass is byte-parallel: the text [0, n_bytes] is cut into tiles of kShTile bytes (one CTA each, 8 bytes per
// thread), whatever the document lengths.
//   count   a tile counts its "unit starts" (char: lead bytes; word: the start of a non-whitespace code point after a
//           whitespace one), ignoring document boundaries, and flags malformed UTF-8 into the status of the document
//           holding the byte.  For every document boundary inside it, the tile stores the unit starts before the boundary.
//   scan    launch_exclusive_scan over the tiles gives G(p), the unit starts before any position p.
//   doc     one thread per document: units m = G(end) - G(start), corrected at the start (the document's first word
//           begins at its first byte whatever precedes it), the O(1) checks at its two ends (a leading continuation byte,
//           a sequence cut by the end), and its shingle count; a second scan gives the token offsets.
//   hash    a tile lists its unit starts; the one at global rank G(p) is unit j = G(p) - base[d] of its document d, and
//           starts shingle j if j is below the document's shingle count.  The thread walks the shingle to find its length
//           and hashes it through a byte reader (hash_core.cuh): no shingle is copied to memory.
// Extra memory: 16 bytes per tile, 28 per document.  Documents with malformed UTF-8 get no shingles.
#pragma once
#include "hash_core.cuh"

namespace dsk {

constexpr int kShThreads = 256;
constexpr int kShTile = kShThreads * 8;

__device__ __forceinline__ uint32_t tbyte(const uint8_t *t, int64_t i) { return __ldg(t + i); }
__device__ __forceinline__ bool is_cont(uint32_t b) { return (b & 0xC0u) == 0x80u; }
// length of the sequence a lead byte opens; 0 for a byte no well-formed sequence starts with (80..C1, F5..FF)
__device__ __forceinline__ int lead_len(uint32_t b) {
    return b < 0x80u ? 1 : b < 0xC2u ? 0 : b < 0xE0u ? 2 : b < 0xF0u ? 3 : b < 0xF5u ? 4 : 0;
}

// a Python whitespace code point starts at i (never at a continuation byte); no byte at or past e is read.
// U+0009-000D, U+001C-0020, U+0085, U+00A0, U+1680, U+2000-200A, U+2028, U+2029, U+202F, U+205F, U+3000
__device__ __forceinline__ bool ws_at(const uint8_t *t, int64_t i, int64_t e) {
    const uint32_t b = tbyte(t, i);
    if (b < 0x80u) return (b >= 0x09u && b <= 0x0Du) || (b >= 0x1Cu && b <= 0x20u);
    if (b != 0xC2u && (b < 0xE1u || b > 0xE3u)) return false;
    if (i + 1 >= e) return false;
    const uint32_t b1 = tbyte(t, i + 1);
    if (b == 0xC2u) return b1 == 0x85u || b1 == 0xA0u;
    if (i + 2 >= e) return false;
    const uint32_t b2 = tbyte(t, i + 2);
    if (b == 0xE1u) return b1 == 0x9Au && b2 == 0x80u;
    if (b == 0xE3u) return b1 == 0x80u && b2 == 0x80u;
    return (b1 == 0x80u && (b2 <= 0x8Au || b2 == 0xA8u || b2 == 0xA9u || b2 == 0xAFu)) || (b1 == 0x81u && b2 == 0x9Fu);
}

// a word starts at i: a non-whitespace code point that is the first in [lo, e) or follows a whitespace one
__device__ __forceinline__ bool word_start(const uint8_t *t, int64_t i, int64_t lo, int64_t e) {
    if (is_cont(tbyte(t, i)) || ws_at(t, i, e)) return false;
    for (int k = 1; k <= 4; ++k) {
        if (i - k < lo) return true;
        if (!is_cont(tbyte(t, i - k))) return ws_at(t, i - k, e);
    }
    return true;   // no lead byte within 4 bytes: only in malformed text
}

template <bool WORD>
__device__ __forceinline__ bool unit_start(const uint8_t *t, int64_t i, int64_t lo, int64_t e) {
    return WORD ? word_start(t, i, lo, e) : !is_cont(tbyte(t, i));
}

// byte i of [lo, hi) is where CPython's strict decoder would fail, reading [lo, hi) as one string: a byte no sequence
// starts with, a lead whose sequence is cut by hi, has a bad second byte (overlong, surrogate, above U+10FFFF) or a
// missing continuation, or a continuation byte no lead covers
__device__ __forceinline__ bool utf8_error(const uint8_t *t, int64_t i, int64_t lo, int64_t hi) {
    const uint32_t b = tbyte(t, i);
    if (b < 0x80u) return false;
    if (is_cont(b)) {
        for (int k = 1; k <= 3; ++k) {
            if (i - k < lo) return true;
            const uint32_t c = tbyte(t, i - k);
            if (!is_cont(c)) return lead_len(c) <= k;
        }
        return true;
    }
    const int len = lead_len(b);
    if (len == 0 || i + len > hi) return true;
    const uint32_t b1 = tbyte(t, i + 1);
    const uint32_t lo1 = b == 0xE0u ? 0xA0u : b == 0xF0u ? 0x90u : 0x80u;
    const uint32_t hi1 = b == 0xEDu ? 0x9Fu : b == 0xF4u ? 0x8Fu : 0xBFu;
    if (b1 < lo1 || b1 > hi1) return true;
    for (int k = 2; k < len; ++k)
        if (!is_cont(tbyte(t, i + k))) return true;
    return false;
}

// the checks utf8_error cannot make for a non-empty document [s, e) read on its own: it starts with a continuation byte,
// or its last sequence is cut by e
__device__ __forceinline__ bool utf8_ends_ok(const uint8_t *t, int64_t s, int64_t e) {
    if (is_cont(tbyte(t, s))) return false;
    for (int k = 1; k <= 3 && e - k >= s; ++k) {
        const uint32_t c = tbyte(t, e - k);
        if (!is_cont(c)) return lead_len(c) <= k;
    }
    return true;
}

// first index in [lo, hi) with a[idx] >= key, else hi (a non-decreasing); all 32 lanes of a warp call it alike
__device__ __forceinline__ int64_t warp_lower_bound(const int64_t *a, int64_t lo, int64_t hi, int64_t key) {
    const int lane = threadIdx.x & 31;
    for (;;) {
        const int64_t len = hi - lo;
        const int64_t step = len > 32 ? (len + 31) / 32 : 1;
        const int64_t idx = lo + lane * step;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, idx >= hi || a[idx] >= key);
        if (step == 1) return m ? lo + __ffs(m) - 1 : hi;
        if (m & 1u) return lo;
        const int f = m ? __ffs(m) - 1 : 32;
        const int64_t nlo = lo + (int64_t)(f - 1) * step + 1;
        hi = min(lo + (int64_t)f * step, hi);
        lo = nlo;
    }
}

// the document holding position p, given that it is one of [a, b]: the largest d there with off[d] <= p
__device__ __forceinline__ int64_t doc_of(const int64_t *off, int64_t a, int64_t b, int64_t p) {
    while (a < b) {
        const int64_t m = a + (b - a + 1) / 2;
        if (off[m] <= p) a = m;
        else b = m - 1;
    }
    return a;
}

// per tile: [rng[0], rng[1]) = the boundaries d (off[d]) inside the tile, [rng[2], rng[3]] = the documents holding its
// bytes in [lo, hi).  Warp 0 searches; the caller synchronises.
__device__ __forceinline__ void tile_ranges(const int64_t *off, int64_t n_docs, int64_t ts, int64_t lo, int64_t hi,
                                            int64_t *rng) {
    if (threadIdx.x >= 32) return;
    const int64_t b_lo = warp_lower_bound(off, 0, n_docs + 1, ts);
    const int64_t b_hi = warp_lower_bound(off, b_lo, n_docs + 1, ts + kShTile);
    const int64_t u_lo = warp_lower_bound(off, 0, n_docs + 1, max(ts, lo) + 1) - 1;
    const int64_t u_hi = warp_lower_bound(off, u_lo < 0 ? 0 : u_lo, n_docs + 1, min(ts + kShTile, hi)) - 1;
    if (threadIdx.x == 0) {
        rng[0] = b_lo; rng[1] = b_hi; rng[2] = u_lo; rng[3] = u_hi;
    }
}

// exclusive scan of one int per thread over the CTA (kShThreads threads); *total = the sum.  Synchronises.
__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int *total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int base = 0, tot = 0;
    for (int w = 0; w < kShThreads / 32; ++w) {
        const int c = s_warp[w];
        if (w < wid) base += c;
        tot += c;
    }
    *total = tot;
    return base + x - v;
}

// unit starts among the thread's 8 bytes of the tile at ts (bit q: byte ts + 8 * thread + q), positions in [lo, hi) only
template <bool WORD>
__device__ __forceinline__ unsigned thread_unit_bits(const uint8_t *t, int64_t ts, int64_t lo, int64_t hi) {
    unsigned bits = 0;
    const int64_t p0 = ts + 8 * (int64_t)threadIdx.x;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const int64_t p = p0 + q;
        if (p >= lo && p < hi && unit_start<WORD>(t, p, lo, hi)) bits |= 1u << q;
    }
    return bits;
}

__device__ __forceinline__ int64_t units_before(const int *s_pre, const uint8_t *s_bits, int64_t q) {
    return s_pre[q >> 3] + __popc(s_bits[q >> 3] & ((1u << (q & 7)) - 1u));
}

__global__ void shingle_offsets_kernel(const int64_t *__restrict__ off, int64_t n_docs, int64_t n_bytes,
                                       int32_t *__restrict__ status, unsigned *__restrict__ bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d <= n_docs; d += stride) {
        status[d] = 0;
        const int64_t o = off[d];
        if (o < 0 || o > n_bytes || (d < n_docs && off[d + 1] < o)) atomicOr(bad, 1u);
    }
}

template <bool WORD>
__global__ void __launch_bounds__(kShThreads) shingle_count_kernel(const uint8_t *__restrict__ t, const int64_t *__restrict__ off,
                                                                   int64_t n_docs, int64_t n_tiles, const unsigned *__restrict__ bad,
                                                                   int32_t *__restrict__ status, int32_t *__restrict__ partial,
                                                                   int64_t *__restrict__ tile_cnt) {
    __shared__ int64_t s_rng[4];
    __shared__ int s_warp[kShThreads / 32];
    __shared__ int s_pre[kShThreads];
    __shared__ uint8_t s_bits[kShThreads];
    if (*bad) return;
    const int64_t lo = off[0], hi = off[n_docs];
    for (int64_t k = blockIdx.x; k < n_tiles; k += gridDim.x) {
        const int64_t ts = k * kShTile;
        if (ts + kShTile <= lo || ts > hi) {          // no byte of a document and no boundary here
            if (threadIdx.x == 0) tile_cnt[k] = 0;
            continue;
        }
        tile_ranges(off, n_docs, ts, lo, hi, s_rng);
        __syncthreads();
        const unsigned bits = thread_unit_bits<WORD>(t, ts, lo, hi);
        const int64_t p0 = ts + 8 * (int64_t)threadIdx.x;
        for (int q = 0; q < 8; ++q) {
            const int64_t p = p0 + q;
            if (p >= lo && p < hi && utf8_error(t, p, lo, hi))
                atomicOr(reinterpret_cast<unsigned *>(status + doc_of(off, s_rng[2], s_rng[3], p)), (unsigned)DSK_SHINGLE_INVALID_UTF8);
        }
        int total;
        const int pre = block_excl_scan(__popc(bits), s_warp, &total);
        s_pre[threadIdx.x] = pre;
        s_bits[threadIdx.x] = (uint8_t)bits;
        if (threadIdx.x == 0) tile_cnt[k] = total;
        __syncthreads();
        for (int64_t d = s_rng[0] + threadIdx.x; d < s_rng[1]; d += kShThreads)
            partial[d] = (int32_t)units_before(s_pre, s_bits, off[d] - ts);
        __syncthreads();
    }
}

template <bool WORD>
__global__ void shingle_doc_kernel(const uint8_t *__restrict__ t, const int64_t *__restrict__ off, int64_t n_docs, int n,
                                   const unsigned *__restrict__ bad, const int64_t *__restrict__ tile_pre,
                                   const int32_t *__restrict__ partial, int32_t *__restrict__ status, int64_t *__restrict__ base,
                                   int64_t *__restrict__ units, int64_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const bool is_bad = *bad != 0;
    const int64_t lo = off[0], hi = off[n_docs];
    for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < n_docs; d += stride) {
        if (is_bad) {
            cnt[d] = 0;
            if (d == 0) atomicOr(reinterpret_cast<unsigned *>(status + n_docs), (unsigned)DSK_SHINGLE_BAD_OFFSETS);
            continue;
        }
        const int64_t s = off[d], e = off[d + 1];
        const int64_t g0 = tile_pre[s / kShTile] + partial[d], g1 = tile_pre[e / kShTile] + partial[d + 1];
        int st = status[d];
        int64_t corr = 0;
        if (s < e) {
            if (!utf8_ends_ok(t, s, e)) st |= DSK_SHINGLE_INVALID_UTF8;
            if (WORD) corr = (int64_t)word_start(t, s, s, e) - (int64_t)word_start(t, s, lo, hi);
        }
        const int64_t m = g1 - g0 + corr;
        base[d] = g0 - corr;
        units[d] = m;
        cnt[d] = st ? 0 : m >= n ? m - n + 1 : m > 0 ? 1 : 0;
        if (st) {
            status[d] = st;
            atomicOr(reinterpret_cast<unsigned *>(status + n_docs), (unsigned)st);
        }
    }
}

// the bytes of a word n-gram: its words, one 0x20 between consecutive ones (the reader is only asked for as many bytes
// as the walk in hash_shingle counted, so the next word always exists where a space is produced)
struct WordReader {
    const uint8_t *t;
    int64_t q, e;
    __device__ __forceinline__ uint32_t next() {
        if (!ws_at(t, q, e)) return tbyte(t, q++);
        while (ws_at(t, q, e)) q += lead_len(tbyte(t, q));
        return 0x20u;
    }
};

// the token of the shingle of n units (n >= 1 of them exist) whose first unit starts at p, in the document ending at e.
// The walk stops at the n-th unit, so whitespace after a document's last word is never scanned.
template <int KIND, bool WORD>
__device__ __forceinline__ uint32_t hash_shingle(const uint8_t *t, int64_t p, int64_t e, int n, uint32_t seed) {
    int64_t q = p;
    if (!WORD) {
        for (int c = 0; c < n && q < e; ++c)
            for (++q; q < e && is_cont(tbyte(t, q)); ++q) {}
        SpanReader rd{t + p};
        return hash32<KIND>(rd, q - p, seed);
    }
    int64_t len = 0;
    int words = 0;
    for (;;) {
        const int64_t s = q;
        while (q < e && !ws_at(t, q, e)) ++q;
        len += q - s;
        if (++words == n) break;
        while (q < e && ws_at(t, q, e)) q += lead_len(tbyte(t, q));
        if (q >= e) break;
        len += 1;
    }
    if (words == 1) {
        SpanReader rd{t + p};
        return hash32<KIND>(rd, len, seed);
    }
    WordReader rd{t, p, e};
    return hash32<KIND>(rd, len, seed);
}

template <int KIND, bool WORD>
__global__ void __launch_bounds__(kShThreads) shingle_hash_kernel(const uint8_t *__restrict__ t, const int64_t *__restrict__ off,
                                                                  int64_t n_docs, int n, int64_t n_tiles, uint32_t seed,
                                                                  const unsigned *__restrict__ bad,
                                                                  const int64_t *__restrict__ tile_pre,
                                                                  const int64_t *__restrict__ base,
                                                                  const int64_t *__restrict__ units,
                                                                  const int64_t *__restrict__ tok_off, uint32_t *__restrict__ out) {
    __shared__ int64_t s_rng[4];
    __shared__ int s_warp[kShThreads / 32];
    __shared__ int s_pre[kShThreads];
    __shared__ uint8_t s_bits[kShThreads];
    __shared__ uint16_t s_items[kShTile];
    __shared__ unsigned s_n;
    if (*bad) return;
    const int64_t lo = off[0], hi = off[n_docs];
    for (int64_t k = blockIdx.x; k < n_tiles; k += gridDim.x) {
        const int64_t ts = k * kShTile;
        if (ts + kShTile <= lo || ts >= hi) continue;   // no unit starts here
        tile_ranges(off, n_docs, ts, lo, hi, s_rng);
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        const unsigned bits = thread_unit_bits<WORD>(t, ts, lo, hi);
        int total;
        const int pre = block_excl_scan(__popc(bits), s_warp, &total);
        s_pre[threadIdx.x] = pre;
        s_bits[threadIdx.x] = (uint8_t)bits;
        // the tile's unit starts, and (word n-grams) the documents whose first word begins at their first byte without a
        // whitespace code point before it in the text: the unit-start count of the count pass skipped those
        for (unsigned b = bits; b; b &= b - 1) s_items[atomicAdd(&s_n, 1u)] = (uint16_t)(8 * threadIdx.x + __ffs(b) - 1);
        if (WORD) {
            for (int64_t d = s_rng[0] + threadIdx.x; d < s_rng[1] && d < n_docs; d += kShThreads) {
                const int64_t s = off[d], e = off[d + 1];
                if (s < e && tok_off[d + 1] > tok_off[d] && word_start(t, s, s, e) && !word_start(t, s, lo, hi))
                    s_items[atomicAdd(&s_n, 1u)] = (uint16_t)(s - ts);
            }
        }
        __syncthreads();
        const int items = (int)s_n;
        for (int i = threadIdx.x; i < items; i += kShThreads) {
            const int64_t q = s_items[i], p = ts + q;
            const int64_t d = doc_of(off, s_rng[2], s_rng[3], p);
            const int64_t t0 = tok_off[d], sd = tok_off[d + 1] - t0;
            if (sd == 0) continue;
            const int64_t j = p == off[d] ? 0 : tile_pre[k] + units_before(s_pre, s_bits, q) - base[d];
            if (j >= sd) continue;
            const int64_t left = units[d] - j;   // units from this one to the document's end
            out[t0 + j] = hash_shingle<KIND, WORD>(t, p, off[d + 1], left < n ? (int)left : n, seed);
        }
        __syncthreads();
    }
}

// ---- workspace and launchers ----------------------------------------------------------------------------------------
struct ShingleWs {
    unsigned *bad;
    int64_t *tile_cnt, *tile_pre, *scratch, *base, *units, *cnt;
    int32_t *partial;
};

static int64_t shingle_tiles(int64_t n_bytes) { return n_bytes / kShTile + 1; }   // positions 0 .. n_bytes, the end included

static ShingleWs shingle_ws(void *ws, int64_t n_docs, int64_t n_bytes, size_t *bytes) {
    const int64_t n_tiles = shingle_tiles(n_bytes);
    const int64_t scan_n = n_tiles > n_docs ? n_tiles : n_docs;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    char *p = static_cast<char *>(ws);
    size_t o = 0;
    ShingleWs w;
    w.bad = reinterpret_cast<unsigned *>(p + o); o += al(sizeof(unsigned));
    w.tile_cnt = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * n_tiles);
    w.tile_pre = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * (n_tiles + 1));
    w.scratch = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * (scan_n / 1024 + 2));
    w.base = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * n_docs);
    w.units = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * n_docs);
    w.cnt = reinterpret_cast<int64_t *>(p + o); o += al(sizeof(int64_t) * n_docs);
    w.partial = reinterpret_cast<int32_t *>(p + o); o += al(sizeof(int32_t) * (n_docs + 1));
    if (bytes) *bytes = o;
    return w;
}

size_t shingle_workspace_bytes(int64_t n_docs, int64_t n_bytes) {
    size_t b;
    shingle_ws(nullptr, n_docs, n_bytes, &b);
    return b;
}

static unsigned shingle_grid(int64_t work, int64_t per_cta, int sm_count) {
    int64_t g = (work + per_cta - 1) / per_cta;
    if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    return (unsigned)(g < 1 ? 1 : g);
}

cudaError_t shingle_count(const uint8_t *text, const int64_t *off, int64_t n_docs, int64_t n_bytes, int word, int n,
                          int64_t *tok_off, int32_t *status, void *ws, int sm_count, cudaStream_t s) {
    const ShingleWs w = shingle_ws(ws, n_docs, n_bytes, nullptr);
    const int64_t n_tiles = shingle_tiles(n_bytes);
    cudaError_t e = cudaMemsetAsync(w.bad, 0, sizeof(unsigned), s);
    if (e != cudaSuccess) return e;
    DSK_LAUNCH(shingle_offsets_kernel, shingle_grid(n_docs + 1, 256, sm_count), 256, 0, s, off, n_docs, n_bytes, status, w.bad);
    const unsigned tg = shingle_grid(n_tiles, 1, sm_count);
    if (word) DSK_LAUNCH(shingle_count_kernel<true>, tg, kShThreads, 0, s, text, off, n_docs, n_tiles, w.bad, status, w.partial, w.tile_cnt);
    else DSK_LAUNCH(shingle_count_kernel<false>, tg, kShThreads, 0, s, text, off, n_docs, n_tiles, w.bad, status, w.partial, w.tile_cnt);
    e = launch_exclusive_scan(w.tile_cnt, n_tiles, w.tile_pre, w.scratch, s);
    if (e != cudaSuccess) return e;
    const unsigned dg = shingle_grid(n_docs, 256, sm_count);
    if (word) DSK_LAUNCH(shingle_doc_kernel<true>, dg, 256, 0, s, text, off, n_docs, n, w.bad, w.tile_pre, w.partial, status, w.base, w.units, w.cnt);
    else DSK_LAUNCH(shingle_doc_kernel<false>, dg, 256, 0, s, text, off, n_docs, n, w.bad, w.tile_pre, w.partial, status, w.base, w.units, w.cnt);
    e = launch_exclusive_scan(w.cnt, n_docs, tok_off, w.scratch, s);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

template <int KIND>
static void launch_shingle_hash_k(unsigned grid, int word, const uint8_t *text, const int64_t *off, int64_t n_docs, int n,
                                  int64_t n_tiles, uint32_t seed, const ShingleWs &w, const int64_t *tok_off, uint32_t *out,
                                  cudaStream_t s) {
    if (word) DSK_LAUNCH((shingle_hash_kernel<KIND, true>), grid, kShThreads, 0, s, text, off, n_docs, n, n_tiles, seed, w.bad, w.tile_pre, w.base, w.units, tok_off, out);
    else DSK_LAUNCH((shingle_hash_kernel<KIND, false>), grid, kShThreads, 0, s, text, off, n_docs, n, n_tiles, seed, w.bad, w.tile_pre, w.base, w.units, tok_off, out);
}

cudaError_t shingle_hash(const uint8_t *text, const int64_t *off, int64_t n_docs, int64_t n_bytes, int word, int n, int kind,
                         uint32_t seed, const int64_t *tok_off, uint32_t *out, void *ws, int sm_count, cudaStream_t s) {
    const ShingleWs w = shingle_ws(ws, n_docs, n_bytes, nullptr);
    const int64_t n_tiles = shingle_tiles(n_bytes);
    const unsigned g = shingle_grid(n_tiles, 1, sm_count);
    if (kind == DSK_HASH_XXH32) launch_shingle_hash_k<DSK_HASH_XXH32>(g, word, text, off, n_docs, n, n_tiles, seed, w, tok_off, out, s);
    else if (kind == DSK_HASH_MURMUR3_32) launch_shingle_hash_k<DSK_HASH_MURMUR3_32>(g, word, text, off, n_docs, n, n_tiles, seed, w, tok_off, out, s);
    else launch_shingle_hash_k<0>(g, word, text, off, n_docs, n, n_tiles, seed, w, tok_off, out, s);
    return cudaGetLastError();
}

}  // namespace dsk
