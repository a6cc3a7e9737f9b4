// emu_tsan_remove_main.cpp -- TEST INFRASTRUCTURE ONLY: the removal-aware self-join (dsk_lsh_remove, then
// dsk_lsh_clusters / dsk_lsh_pairs_*) of the emulated library under ThreadSanitizer.
//   g++ -std=c++17 -O1 -g -pthread -fsanitize=thread -DDSK_EMU -Itests/emu tests/emu/emu_capi.cpp tests/emu/emu_tsan_remove_main.cpp
// One big component with removed members spread through it: the remaining members hook roots with atomicCAS while other
// host threads (the emulated lanes) walk parent paths and read the removal bitmap; a racing access that is not atomic is a
// data race TSan reports.  The results are checked against brute-force pairs of the remaining documents and a serial
// union-find (removed documents: label -1).  Run with TSAN_OPTIONS=history_size=7 (see emu_tsan_main.cpp).
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/dsk.h"

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() {
    rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
    return rng_state;
}

static int find(std::vector<int32_t> &p, int x) {
    while (p[x] != x) x = p[x];
    return x;
}

struct Case {
    int k, b, r;
    int64_t n;
    std::vector<uint32_t> sig;
    std::vector<char> gone;
    // brute force: every pair d < i of remaining documents with an equal band tuple, and its count of equal positions
    std::vector<int64_t> pi, pd;
    std::vector<int32_t> peq;
    void pairs() {
        for (int64_t i = 0; i < n; ++i)
            for (int64_t d = 0; d < i; ++d) {
                if (gone[i] || gone[d]) continue;
                bool cand = false;
                for (int j = 0; j < b && !cand; ++j) {
                    bool eq = true;
                    for (int q = 0; q < r; ++q) eq = eq && sig[i * k + j * r + q] == sig[d * k + j * r + q];
                    cand = eq;
                }
                if (!cand) continue;
                int e = 0;
                for (int q = 0; q < k; ++q) e += sig[i * k + q] == sig[d * k + q];
                pi.push_back(i); pd.push_back(d); peq.push_back(e);
            }
    }
    std::vector<int32_t> labels(int min_count) const {
        std::vector<int32_t> p(n);
        for (int64_t i = 0; i < n; ++i) p[i] = (int32_t)i;
        for (size_t e = 0; e < pi.size(); ++e) {
            if (peq[e] < min_count) continue;
            const int a = find(p, (int)pi[e]), c = find(p, (int)pd[e]);
            if (a != c) p[a > c ? a : c] = a > c ? c : a;
        }
        for (int64_t i = 0; i < n; ++i) p[i] = gone[i] ? -1 : find(p, (int)i);
        return p;
    }
};

// n documents, the first `star` of them with one tuple in band 0 (one big component); every third of those removed, and
// a few others; the other values drawn from `vals`
static Case make(int64_t n, int64_t star, int vals) {
    Case c{32, 8, 4, n, {}, {}, {}, {}, {}};
    c.sig.resize((size_t)n * c.k);
    for (auto &v : c.sig) v = (uint32_t)(rnd() % vals);
    for (int64_t i = 0; i < star; ++i)
        for (int q = 0; q < c.r; ++q) c.sig[i * c.k + q] = 7u + q;
    c.gone.assign(n, 0);
    for (int64_t i = 0; i < star; i += 3) c.gone[i] = 1;
    for (int64_t i = star; i < n; i += 7) c.gone[i] = 1;
    c.pairs();
    return c;
}

static dsk_lsh *index_of(const Case &c) {
    dsk_lsh *ix = nullptr;
    if (dsk_lsh_create(c.k, c.b, c.r, c.n, 0, &ix) != DSK_OK) return nullptr;
    const int64_t h = c.n / 3;   // two batches
    dsk_lsh_insert(ix, c.sig.data(), h, nullptr);
    dsk_lsh_insert(ix, c.sig.data() + h * c.k, c.n - h, nullptr);
    std::vector<int32_t> ids;
    for (int64_t i = 0; i < c.n; ++i)
        if (c.gone[i]) ids.push_back((int32_t)i);
    int64_t status[2] = {0, 0};
    if (dsk_lsh_remove(ix, ids.data(), (int64_t)ids.size(), status, nullptr) != DSK_OK || status[0] || status[1]) {
        dsk_lsh_destroy(ix);
        return nullptr;
    }
    return ix;
}

static bool clusters_ok(const Case &c, dsk_lsh *ix, int min_count) {
    std::vector<int32_t> got(c.n, -7);
    return dsk_lsh_clusters(ix, min_count, got.data(), nullptr) == DSK_OK && got == c.labels(min_count);
}

int main() {
    int bad = 0;
    {   // linear link path: 500 of 700 documents in one bucket of band 0, a third of them removed
        Case c = make(700, 500, 3);
        dsk_lsh *ix = index_of(c);
        const bool ok = ix && clusters_ok(c, ix, 0);
        printf("clusters with removals, min_count 0: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        dsk_lsh_destroy(ix);
    }
    {   // pair walk: unions straight from the walk, and the count -> scan -> fill of the same pairs
        Case c = make(140, 90, 3);
        dsk_lsh *ix = index_of(c);
        bool ok = ix && clusters_ok(c, ix, 14);
        printf("clusters with removals, min_count 14: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        ok = ix && clusters_ok(c, ix, 0);
        printf("clusters of the same index, min_count 0: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        std::vector<int64_t> counts(c.n), ptr(c.n + 1), scratch(c.n / 1024 + 2);
        ok = ix && dsk_lsh_pairs_count(ix, 14, counts.data(), nullptr) == DSK_OK &&
             dsk_exclusive_scan(counts.data(), c.n, ptr.data(), scratch.data(), nullptr) == DSK_OK;
        std::vector<int32_t> idx(ok ? ptr[c.n] + 1 : 1), eq(idx.size());
        ok = ok && dsk_lsh_pairs_fill(ix, 14, ptr.data(), idx.data(), eq.data(), nullptr) == DSK_OK;
        std::vector<int64_t> want(c.n * c.n, -1), got(c.n * c.n, -1);
        for (size_t e = 0; e < c.pi.size(); ++e)
            if (c.peq[e] >= 14) want[c.pi[e] * c.n + c.pd[e]] = c.peq[e];
        for (int64_t i = 0; ok && i < c.n; ++i)
            for (int64_t p = ptr[i]; p < ptr[i + 1]; ++p) {
                ok = idx[p] >= 0 && idx[p] < i && got[i * c.n + idx[p]] < 0;
                if (ok) got[i * c.n + idx[p]] = eq[p];
            }
        ok = ok && got == want;
        printf("pairs with removals, min_count 14: %s\n", ok ? "identical" : "MISMATCH");
        bad += !ok;
        dsk_lsh_destroy(ix);
    }
    return bad ? 1 : 0;
}
