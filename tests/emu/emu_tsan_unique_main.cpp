// emu_tsan_unique_main.cpp -- TEST INFRASTRUCTURE ONLY: dsk_lsh_unique_count / dsk_lsh_unique_commit of the emulated
// library under ThreadSanitizer.
//   g++ -std=c++17 -O1 -g -pthread -fsanitize=thread -DDSK_EMU -Itests/emu tests/emu/emu_capi.cpp tests/emu/emu_tsan_unique_main.cpp
// The greedy resolution reads the statuses of a row's earlier partners while other host threads (the emulated lanes)
// decide those rows and write theirs: every such access must be one of the relaxed atomics, or TSan reports a data race.
// The batches hold drift chains (row i matches i - 1 only), so most decisions wait for another thread's, over many rounds
// of the resolving CTA.  Results are checked against the serial loop over brute-force candidates.  Run with
// TSAN_OPTIONS=history_size=7 (see emu_tsan_main.cpp).
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/dsk.h"

static uint64_t rng_state = 0x2545F4914F6CDD1Dull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
    return rng_state;
}

constexpr int K = 32, B = 8, R = 4;

static bool candidate(const uint32_t *a, const uint32_t *c) {
    for (int j = 0; j < B; ++j) {
        bool eq = true;
        for (int q = 0; q < R; ++q) eq = eq && a[j * R + q] == c[j * R + q];
        if (eq) return true;
    }
    return false;
}

static int count_eq(const uint32_t *a, const uint32_t *c) {
    int e = 0;
    for (int q = 0; q < K; ++q) e += a[q] == c[q];
    return e;
}

// `chains` drift chains of `len` rows each, interleaved, plus `noise` unrelated rows and a few exact copies
static std::vector<uint32_t> make_batch(int chains, int len, int noise) {
    std::vector<uint32_t> sig;
    std::vector<std::vector<uint32_t>> vals(chains * B, std::vector<uint32_t>((len / 2 + 2) * R));
    for (auto &v : vals)
        for (auto &x : v) x = (uint32_t)rnd();
    for (int i = 0; i < len; ++i)
        for (int c = 0; c < chains; ++c) {
            for (int j = 0; j < B; ++j) {
                const int g = (i + (j & 1)) / 2;   // rows i and i + 1 share the even bands for even i, the odd ones for odd i
                for (int q = 0; q < R; ++q) sig.push_back(vals[c * B + j][g * R + q]);
            }
            for (int q = B * R; q < K; ++q) sig.push_back((uint32_t)rnd());
        }
    for (int i = 0; i < noise; ++i)
        for (int q = 0; q < K; ++q) sig.push_back((uint32_t)rnd());
    const size_t rows = sig.size() / K;
    for (int i = 0; i < 20; ++i) {   // exact copies of earlier rows
        const size_t src = rnd() % rows;
        for (int q = 0; q < K; ++q) sig.push_back(sig[src * K + q]);
    }
    return sig;
}

// the serial loop: kept flags, matches and eq against `held` (the index's rows) and the kept rows before each row
static void serial(const std::vector<uint32_t> &held0, const std::vector<uint32_t> &batch, int min_count,
                   std::vector<uint8_t> &kept, std::vector<int32_t> &match, std::vector<int32_t> &eq) {
    std::vector<uint32_t> held = held0;
    const int64_t n = (int64_t)batch.size() / K;
    kept.assign(n, 0);
    match.assign(n, -1);
    eq.assign(n, -1);
    for (int64_t j = 0; j < n; ++j) {
        const uint32_t *row = batch.data() + j * K;
        const int64_t nd = (int64_t)held.size() / K;
        for (int64_t d = 0; d < nd; ++d) {
            const uint32_t *dr = held.data() + d * K;
            if (!candidate(row, dr)) continue;
            const int e = count_eq(row, dr);
            if (e >= min_count && e > eq[j]) { eq[j] = e; match[j] = (int32_t)d; }   // ascending d: ties keep the smaller
        }
        if (match[j] < 0) {
            kept[j] = 1;
            held.insert(held.end(), row, row + K);
        }
    }
}

static bool run(dsk_lsh *ix, const std::vector<uint32_t> &held, const std::vector<uint32_t> &batch, int min_count) {
    const int64_t n = (int64_t)batch.size() / K;
    const size_t ws_bytes = dsk_lsh_unique_workspace_size(ix, n);
    std::vector<uint64_t> ws(ws_bytes / 8 + 2);
    std::vector<int64_t> counts(n), ptr(n + 1), scratch(n / 1024 + 2);
    if (dsk_lsh_unique_count(ix, batch.data(), n, min_count, ws.data(), ws_bytes, counts.data(), nullptr) != DSK_OK ||
        dsk_exclusive_scan(counts.data(), n, ptr.data(), scratch.data(), nullptr) != DSK_OK)
        return false;
    std::vector<int32_t> pidx(ptr[n] + 1), peq(ptr[n] + 1), match(n), eq(n);
    std::vector<uint8_t> kept(n);
    int64_t inserted = -1;
    if (dsk_lsh_unique_commit(ix, batch.data(), n, min_count, ws.data(), ws_bytes, ptr.data(), pidx.data(), peq.data(),
                              kept.data(), match.data(), eq.data(), &inserted, nullptr) != DSK_OK)
        return false;
    std::vector<uint8_t> w_kept;
    std::vector<int32_t> w_match, w_eq;
    serial(held, batch, min_count, w_kept, w_match, w_eq);
    int64_t m = 0;
    for (auto x : w_kept) m += x;
    return kept == w_kept && match == w_match && eq == w_eq && inserted == m;
}

int main() {
    int bad = 0;
    const std::vector<uint32_t> held = make_batch(2, 6, 30);   // the index: short chains and unrelated rows
    {   // one long chain (many rounds), into an empty index
        dsk_lsh *ix = nullptr;
        const std::vector<uint32_t> batch = make_batch(1, 300, 20);
        bool ok = dsk_lsh_create(K, B, R, 4000, 0, &ix) == DSK_OK && run(ix, {}, batch, 0);
        printf("one chain of 300, no threshold: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        dsk_lsh_destroy(ix);
    }
    {   // many interleaved chains against an index, with a threshold (eq >= 16 between neighbours)
        dsk_lsh *ix = nullptr;
        const std::vector<uint32_t> batch = make_batch(8, 60, 40);
        bool ok = dsk_lsh_create(K, B, R, 4000, 0, &ix) == DSK_OK &&
                  dsk_lsh_insert(ix, held.data(), (int64_t)held.size() / K, nullptr) == DSK_OK &&
                  run(ix, held, batch, 16);
        printf("eight chains of 60 against an index, min_count 16: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        // the same batch again: everything is a duplicate of what the first call kept or of the index
        std::vector<uint32_t> now = held;
        {
            std::vector<uint8_t> k0;
            std::vector<int32_t> m0, e0;
            serial(held, batch, 16, k0, m0, e0);
            for (size_t j = 0; j < k0.size(); ++j)
                if (k0[j]) now.insert(now.end(), batch.begin() + j * K, batch.begin() + (j + 1) * K);
        }
        ok = ok && run(ix, now, batch, 16);
        printf("the same batch again: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        dsk_lsh_destroy(ix);
    }
    return bad ? 1 : 0;
}
