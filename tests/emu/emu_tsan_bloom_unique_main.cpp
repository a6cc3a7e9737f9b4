// emu_tsan_bloom_unique_main.cpp -- TEST INFRASTRUCTURE ONLY: dsk_bloom_unique of the emulated library under
// ThreadSanitizer.
//   g++ -std=c++17 -O1 -g -pthread -fsanitize=thread -DDSK_EMU -Itests/emu tests/emu/emu_capi.cpp tests/emu/emu_tsan_bloom_unique_main.cpp
// The resolution reads the statuses of the earlier setters of a row's probe bits while other host threads (the emulated
// lanes) decide those rows and write theirs: every such access must be one of the relaxed atomics, or TSan reports a data
// race.  The batches hold band-level drift chains (row i copies one band of row i - 1), so most decisions wait for another
// thread's, over many rounds of the resolving CTA, plus exact copies.  Results are checked against the serial loop over a
// host model of the tables.  Run with TSAN_OPTIONS=history_size=7 (see emu_tsan_main.cpp).
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/dsk.h"

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
    return rng_state;
}

constexpr int K = 32, B = 4, R = 8, H = 3;

static uint64_t mix(uint64_t h) {
    h ^= h >> 33; h *= 0xFF51AFD7ED558CCDull; h ^= h >> 33; h *= 0xC4CEB9FE1A85EC53ull; h ^= h >> 33;
    return h;
}

// the probe positions of band j of a row (the library's documented scheme: key = sum % (2^61 - 1), double hashing)
static void positions(const uint32_t *row, int j, uint64_t n_bits, uint64_t *pos) {
    uint64_t x = 0;
    for (int q = 0; q < R; ++q) x += row[j * R + q];
    x %= (1ull << 61) - 1;
    const uint64_t h1 = mix(x ^ 0x9E3779B97F4A7C15ull), h2 = mix(x + 0xD6E8FEB86659FD93ull) | 1ull;
    for (int q = 0; q < H; ++q) pos[q] = (h1 + (uint64_t)q * h2) % n_bits;
}

// the serial loop over a host copy of the tables
static std::vector<uint8_t> serial(std::vector<uint32_t> &tab, uint64_t words, uint64_t n_bits, const std::vector<uint32_t> &sig) {
    const size_t n = sig.size() / K;
    std::vector<uint8_t> keep(n, 0);
    uint64_t pos[H];
    for (size_t i = 0; i < n; ++i) {
        const uint32_t *row = sig.data() + i * K;
        bool hit = false;
        for (int j = 0; j < B && !hit; ++j) {
            positions(row, j, n_bits, pos);
            bool all = true;
            for (int q = 0; q < H; ++q) all = all && ((tab[j * words + (pos[q] >> 5)] >> (pos[q] & 31)) & 1u);
            hit = all;
        }
        if (hit) continue;
        keep[i] = 1;
        for (int j = 0; j < B; ++j) {
            positions(row, j, n_bits, pos);
            for (int q = 0; q < H; ++q) tab[j * words + (pos[q] >> 5)] |= 1u << (pos[q] & 31);
        }
    }
    return keep;
}

// `chains` band-level drift chains of `len` rows, interleaved, then unrelated rows and exact copies of earlier rows
static std::vector<uint32_t> make_batch(int chains, int len, int noise) {
    std::vector<uint32_t> sig;
    std::vector<std::vector<uint32_t>> prev(chains, std::vector<uint32_t>(K));
    for (auto &p : prev)
        for (auto &x : p) x = (uint32_t)rnd();
    for (int i = 0; i < len; ++i)
        for (int c = 0; c < chains; ++c) {
            std::vector<uint32_t> row(K);
            for (auto &x : row) x = (uint32_t)rnd();
            const int t = i % B;
            for (int q = 0; q < R; ++q) row[t * R + q] = prev[c][t * R + q];
            prev[c] = row;
            sig.insert(sig.end(), row.begin(), row.end());
        }
    for (int i = 0; i < noise * K; ++i) sig.push_back((uint32_t)rnd());
    const size_t rows = sig.size() / K;
    for (int i = 0; i < 20; ++i) {
        const size_t src = rnd() % rows;
        for (int q = 0; q < K; ++q) sig.push_back(sig[src * K + q]);
    }
    return sig;
}

static int run(int chains, int len, int noise, uint64_t n_bits) {
    const uint64_t words = (n_bits + 31) / 32;
    const std::vector<uint32_t> sig = make_batch(chains, len, noise);
    const int64_t n = (int64_t)sig.size() / K;
    std::vector<uint32_t> tab(B * words, 0), model(B * words, 0);
    const std::vector<uint8_t> want = serial(model, words, n_bits, sig);
    const size_t need = dsk_bloom_unique_workspace_size(n, K, B, R, H);
    std::vector<uint64_t> ws(need / 8 + 2);
    std::vector<uint8_t> keep(n, 7);
    if (dsk_bloom_unique(sig.data(), n, K, B, R, tab.data(), words, n_bits, H, ws.data(), need, keep.data(), nullptr) != 0) {
        printf("dsk_bloom_unique failed: %s\n", dsk_last_error());
        return 1;
    }
    if (keep != want || tab != model) {
        printf("MISMATCH chains=%d len=%d\n", chains, len);
        return 1;
    }
    int kept = 0;
    for (uint8_t k : keep) kept += k;
    printf("identical: %lld rows, %d kept\n", (long long)n, kept);
    return 0;
}

int main() {
    int rc = run(1, 300, 40, 1ull << 20);   // one chain: a round per row in the resolving CTA
    rc |= run(4, 60, 100, 4099);             // several chains among noise in a small table
    return rc;
}
