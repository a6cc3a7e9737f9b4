"""GpuLSH(weighted=True): a device-resident MinHashLSH over WeightedMinHash signatures.

The reference's MinHashLSH takes WeightedMinHash objects as well (test/test_lsh.py's TestWeightedMinHashLSH): a band key
is the byteswapped bytes of r (k, t) int64 pairs (lsh.py:344, :537-538) and the similarity is WeightedMinHash.jaccard, the
fraction of samples whose (k, t) pairs are equal (weighted_minhash.py:55-60).  The index packs sample j into words 2j (k
as uint32) and 2j + 1 (t as int32), bands over 2r words, and counts eq per SAMPLE whose two words both agree.

The oracle is oracle_np.DictLSH over the [ss, 2] rows (with test_lsh_remove.py's MinHashLSH.remove), oracle_np.wmh_jaccard
and scipy's connected components; tests/golden/lsh_weighted.npz (oracle/gen_golden_lsh_weighted.py) pins it to the
reference.  Two backends, as in test_lsh_query_jaccard.py: ``emu``, the whole library on the emulation shim driven through
its C-ABI (rows packed by the product's own packer on the CPU), and ``gpu``, the Python API on the H100.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402
from test_lsh_self_join import _aligned, _components, _p  # noqa: E402
from test_lsh_remove import _DictLSH  # noqa: E402

DSK_OK, DSK_ERR_INVALID, DSK_ERR_ALIGN = 0, 1, 4
CONFIGS = ("a", "b", "c")


def _mc(min_jaccard, ss):
    from datasketch_b200.lsh import _jaccard_min_count
    return _jaccard_min_count(min_jaccard, ss)


def _pack_cpu(rows, ss):
    """The product's packer, run on the CPU: [N, ss, 2] (k, t) -> [N, 2 * ss] u32."""
    from datasketch_b200.lsh import _pack_weighted
    return _pack_weighted(rows, ss, "cpu").numpy().view(np.uint32)


def _unpack(words):
    """[N, 2 * ss] u32 words -> [N, ss, 2] int64 (k, t): every word pattern is a valid packing."""
    w = np.ascontiguousarray(words, dtype=np.uint32)
    return np.stack([w[:, 0::2].astype(np.int64), w[:, 1::2].view(np.int32).astype(np.int64)], axis=-1)


# ---- backends ----------------------------------------------------------------------------------------------------------
class _EmuW:
    """The emulated library through its C-ABI: a weighted handle, rows packed on the CPU."""

    def __init__(self, lib, ss, b, r, capacity):
        self.lib, self.ss, self.n = lib, ss, 0
        self.h = ctypes.c_void_p()
        assert lib.dsk_lsh_create_weighted(ss, b, r, capacity, 0, ctypes.byref(self.h)) == 0, lib.dsk_last_error()

    def _rows(self, rows):
        return _aligned(_pack_cpu(rows, self.ss))

    def __len__(self):
        size = ctypes.c_int64()
        assert self.lib.dsk_lsh_size(self.h, ctypes.byref(size), None) == 0
        return size.value

    def insert(self, rows):
        w = self._rows(rows)
        assert self.lib.dsk_lsh_insert(self.h, _p(w), len(w), None) == 0, self.lib.dsk_last_error()

    def query(self, rows):
        lib, w = self.lib, self._rows(rows)
        nq = len(w)
        counts, ptr = np.zeros(nq + 1, dtype=np.int64), np.zeros(nq + 1, dtype=np.int64)
        scratch = np.zeros(nq // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_query_count(self.h, _p(w), nq, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), nq, _p(ptr), _p(scratch), None) == 0
        idx = np.full(max(int(ptr[-1]), 1), -1, dtype=np.int32)
        assert lib.dsk_lsh_query_fill(self.h, _p(w), nq, _p(ptr), _p(idx), None) == 0, lib.dsk_last_error()
        return ptr, idx[:int(ptr[-1])]

    def query_jaccard(self, rows, t=None):
        lib, w, mc = self.lib, self._rows(rows), _mc(t, self.ss)
        nq = len(w)
        counts, ptr = np.full(nq + 1, -7, dtype=np.int64), np.zeros(nq + 1, dtype=np.int64)
        scratch = np.zeros(nq // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_query_jaccard_count(self.h, _p(w), nq, mc, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), nq, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        idx, eq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_query_jaccard_fill(self.h, _p(w), nq, mc, _p(ptr), _p(idx), _p(eq), None) == 0
        return ptr, idx[:m], eq[:m]

    def query_best(self, rows, t=None):
        lib, w, mc = self.lib, self._rows(rows), _mc(t, self.ss)
        nq = len(w)
        idx, eq = np.full(max(nq, 1), -7, dtype=np.int32), np.full(max(nq, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_query_best(self.h, _p(w), nq, mc, _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return idx[:nq], eq[:nq]

    def pairs(self, t=None):
        lib, n, mc = self.lib, len(self), _mc(t, self.ss)
        counts, ptr = np.zeros(n + 1, dtype=np.int64), np.zeros(n + 1, dtype=np.int64)
        scratch = np.zeros(n // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_pairs_count(self.h, mc, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), n, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        idx, eq = np.full(max(m, 1), -1, dtype=np.int32), np.full(max(m, 1), -1, dtype=np.int32)
        assert lib.dsk_lsh_pairs_fill(self.h, mc, _p(ptr), _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return ptr, idx[:m], eq[:m]

    def clusters(self, t=None):
        n = len(self)
        labels = np.full(max(n, 1), -7, dtype=np.int32)
        assert self.lib.dsk_lsh_clusters(self.h, _mc(t, self.ss), _p(labels), None) == 0, self.lib.dsk_last_error()
        return labels[:n]

    def remove(self, docs):
        d = _aligned(np.asarray(docs, dtype=np.int32).reshape(-1))
        status = np.zeros(2, dtype=np.int64)
        assert self.lib.dsk_lsh_remove(self.h, _p(d), len(d), _p(status), None) == 0, self.lib.dsk_last_error()

    def compact(self):
        lib, n = self.lib, len(self)
        ws = _aligned(np.zeros(max(int(lib.dsk_lsh_compact_workspace_size(self.h)), 1), dtype=np.uint8))
        remap = np.full(max(n, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_compact(self.h, _p(remap), _p(ws), ws.nbytes, None) == 0, lib.dsk_last_error()
        return remap[:n]

    def insert_unique(self, rows, t=None):
        lib, w, mc = self.lib, self._rows(rows), _mc(t, self.ss)
        n = len(w)
        ws_bytes = int(lib.dsk_lsh_unique_workspace_size(self.h, n))
        ws = _aligned(np.zeros(max(ws_bytes, 1), dtype=np.uint8))
        counts, ptr = np.full(n + 1, -7, dtype=np.int64), np.zeros(n + 1, dtype=np.int64)
        scratch = np.zeros(n // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_unique_count(self.h, _p(w), n, mc, _p(ws), ws_bytes, _p(counts), None) == 0, \
            lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), n, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        pidx, peq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        kept = np.full(max(n, 1), 7, dtype=np.uint8)
        match, eq = np.full(max(n, 1), -7, dtype=np.int32), np.full(max(n, 1), -7, dtype=np.int32)
        ins = ctypes.c_int64(-7)
        assert lib.dsk_lsh_unique_commit(self.h, _p(w), n, mc, _p(ws), ws_bytes, _p(ptr), _p(pidx), _p(peq), _p(kept),
                                         _p(match), _p(eq), ctypes.byref(ins), None) == 0, lib.dsk_last_error()
        return kept[:n].astype(bool), match[:n], eq[:n]

    def close(self):
        self.lib.dsk_lsh_destroy(self.h)


class _GpuW:
    """The Python API on the H100: GpuLSH(weighted=True) with [N, ss, 2] int64 numpy rows."""

    def __init__(self, dsk, ss, b, r, capacity):
        self.ix = dsk.GpuLSH(num_perm=ss, params=(b, r), capacity=capacity, weighted=True)

    def __len__(self):
        return len(self.ix)

    def __getattr__(self, name):
        return getattr(self.ix, name)

    def pairs(self, t=None):
        return self.ix.candidate_pairs(t)

    def clusters(self, t=None):
        return self.ix.duplicate_clusters(t)

    def insert_unique(self, rows, t=None):
        return self.ix.insert_unique(rows, t)

    def close(self):
        pass


class _Emu:
    name = "emu"

    def __init__(self, lib):
        self.lib = lib

    def index(self, ss, b, r, capacity):
        return _EmuW(self.lib, ss, b, r, capacity)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk

    def index(self, ss, b, r, capacity):
        return _GpuW(self.dsk, ss, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
def _eq(x, y):
    return int(np.count_nonzero(np.all(x == y, axis=1)))


def _oracle(rows, alive, ss, b, r):
    ref = _DictLSH(ss, b, r)
    for i, row in enumerate(rows):
        ref.insert(i, row)
    for i in np.flatnonzero(~alive).tolist():
        ref.remove(i)
    return ref


def _want(ref, rows, qs, t):
    """Per query {d: eq} over DictLSH.query with WeightedMinHash.jaccard (oracle_np.wmh_jaccard) >= t (None: all)."""
    return [{d: _eq(q, rows[d]) for d in ref.query(q) if t is None or o.wmh_jaccard(q, rows[d]) >= t} for q in qs]


def _got(ptr, idx, eq):
    assert ptr[0] == 0 and np.all(np.diff(ptr) >= 0) and ptr[-1] == len(idx) == len(eq)
    out = []
    for q in range(len(ptr) - 1):
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        d = dict(zip(idx[sl].tolist(), eq[sl].tolist()))
        assert len(d) == ptr[q + 1] - ptr[q]
        out.append(d)
    return out


def _lists(ptr, idx):
    return [sorted(idx[ptr[q]:ptr[q + 1]].tolist()) for q in range(len(ptr) - 1)]


def _check_queries(ix, rows, qs, ss, b, r, thresholds, alive=None):
    alive = np.ones(len(rows), dtype=bool) if alive is None else alive
    ref = _oracle(rows, alive, ss, b, r)
    for t in thresholds:
        want = _want(ref, rows, qs, t)
        assert _got(*ix.query_jaccard(qs, t)) == want, t
        bi, bq = ix.query_best(qs, t)
        best = [min(((-e, d) for d, e in w.items()), default=(1, -1)) for w in want]
        assert list(zip(bi.tolist(), bq.tolist())) == [(d, -e) if d >= 0 else (-1, -1) for e, d in best], t
        if t is None:
            assert _lists(*ix.query(qs)) == [sorted(w) for w in want]
    return ref


def _check_pairs(ix, rows, ss, b, r, thresholds, alive=None):
    alive = np.ones(len(rows), dtype=bool) if alive is None else alive
    ref = _oracle(rows, alive, ss, b, r)
    n = len(rows)
    for t in thresholds:
        want = {(i, d): e for i in np.flatnonzero(alive).tolist()
                for d, e in _want(ref, rows, rows[i:i + 1], t)[0].items() if d < i}
        ptr, idx, eq = ix.pairs(t)
        rows_i = np.repeat(np.arange(n), np.diff(ptr))
        got = dict(zip(zip(rows_i.tolist(), idx.tolist()), eq.tolist()))
        assert len(got) == len(idx) and got == want, t
        labels = _components(n, want).astype(np.int64) if n else np.zeros(0, dtype=np.int64)
        labels[~alive] = -1
        assert np.array_equal(np.asarray(ix.clusters(t), dtype=np.int64), labels), t


def _golden(golden, cfg):
    g = golden("lsh_weighted")
    return {k[len(cfg) + 1:]: g[k] for k in g.files if k.startswith(cfg + "_")}


def _csr_lists(g, which):
    return _lists(g[which + "_ptr"], g[which + "_idx"])


# ---- the reference (tests/golden/lsh_weighted.npz) ---------------------------------------------------------------------
@pytest.mark.parametrize("cfg", CONFIGS)
def test_oracle_is_the_reference(golden, cfg):
    """DictLSH over the [ss, 2] rows and wmh_jaccard give the reference's query lists, jaccards, filtered lists, dedup
    loop and lists after removal."""
    g = _golden(golden, cfg)
    b, r, ss = g["params"].tolist()
    hv, qhv = g["hv"], g["qhv"]
    ref = _oracle(hv, np.ones(len(hv), dtype=bool), ss, b, r)
    for tag, qs in (("q", qhv), ("s", hv[:len(g["s_ptr"]) - 1])):
        lists = [sorted(ref.query(q)) for q in qs]
        assert lists == _csr_lists(g, tag)
        assert [o.wmh_jaccard(q, hv[d]) for q, x in zip(qs, lists) for d in x] == g[tag + "_jaccard"].tolist()
        for j, t in enumerate(g["thresholds"].tolist()):
            assert [sorted(w) for w in _want(ref, hv, qs, t)] == _csr_lists(g, "%s_kept%d" % (tag, j))
    for j, t in enumerate(g["thresholds"].tolist()):
        ref, held, kept = _oracle(hv, np.ones(len(hv), dtype=bool), ss, b, r), list(hv), []
        for q in qhv:
            if not [d for d in ref.query(q) if o.wmh_jaccard(q, held[d]) >= t]:
                ref.insert(len(held), q)
                held.append(q)
                kept.append(1)
            else:
                kept.append(0)
        assert kept == g["uniq%d_kept" % j].tolist()
    alive = np.ones(len(hv), dtype=bool)
    alive[g["removed"]] = False
    ref = _oracle(hv, alive, ss, b, r)
    assert [sorted(ref.query(q)) for q in qhv] == _csr_lists(g, "rq")
    assert sum(len(x) for x in _csr_lists(g, "q_kept1")) > 0 and g["uniq1_kept"].any() or cfg == "c"


@pytest.mark.parametrize("cfg", CONFIGS)
def test_golden_queries_pairs_and_clusters(be, golden, cfg):
    """The reference's query lists and WeightedMinHash.jaccard (= eq / ss) for held-out and indexed rows, the filtered
    lists, query_best, and the self-join and clusters against the oracle."""
    g = _golden(golden, cfg)
    b, r, ss = g["params"].tolist()
    hv, qhv = g["hv"], g["qhv"]
    ix = be.index(ss, b, r, len(hv))
    try:
        ix.insert(hv[:len(hv) // 2])
        ix.insert(hv[len(hv) // 2:])
        for tag, qs in (("q", qhv), ("s", hv[:len(g["s_ptr"]) - 1])):
            got = _got(*ix.query_jaccard(qs))
            assert [sorted(x) for x in got] == _csr_lists(g, tag)
            assert [x[d] / float(ss) for x in got for d in sorted(x)] == g[tag + "_jaccard"].tolist()
            for j, t in enumerate(g["thresholds"].tolist()):
                assert [sorted(x) for x in _got(*ix.query_jaccard(qs, t))] == _csr_lists(g, "%s_kept%d" % (tag, j))
        _check_queries(ix, hv, qhv, ss, b, r, (None,) + tuple(g["thresholds"].tolist()))
        _check_pairs(ix, hv, ss, b, r, (None,) + tuple(g["thresholds"].tolist()))
    finally:
        ix.close()


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("j", [0, 1])
def test_golden_insert_unique(be, golden, cfg, j):
    """insert_unique of the held-out batch equals the reference's streaming dedup loop: kept rows, best match and its
    WeightedMinHash.jaccard; the index then answers as one holding the loop's documents."""
    g = _golden(golden, cfg)
    b, r, ss = g["params"].tolist()
    hv, qhv = g["hv"], g["qhv"]
    t = g["thresholds"].tolist()[j]
    ix = be.index(ss, b, r, len(hv) + len(qhv))
    try:
        ix.insert(hv)
        kept, match, eq = ix.insert_unique(qhv, t)
        assert kept.tolist() == g["uniq%d_kept" % j].astype(bool).tolist()
        assert match.tolist() == g["uniq%d_match" % j].tolist()
        assert [e / float(ss) if e >= 0 else -1.0 for e in eq.tolist()] == g["uniq%d_jaccard" % j].tolist()
        rows = np.concatenate([hv, qhv[kept]])
        assert len(ix) == len(rows)
        _check_queries(ix, rows, qhv, ss, b, r, (None, t))
    finally:
        ix.close()


@pytest.mark.parametrize("cfg", CONFIGS)
def test_golden_remove_then_compact(be, golden, cfg):
    """After removing the fixture's 20 keys the query lists are the reference's; pairs and clusters are the oracle's with
    the removed documents labelled -1; after compact() everything is the same through remap."""
    g = _golden(golden, cfg)
    b, r, ss = g["params"].tolist()
    hv, qhv = g["hv"], g["qhv"]
    ix = be.index(ss, b, r, len(hv))
    try:
        ix.insert(hv)
        ix.remove(g["removed"])
        alive = np.ones(len(hv), dtype=bool)
        alive[g["removed"]] = False
        assert _lists(*ix.query(qhv)) == _csr_lists(g, "rq")
        assert _lists(*ix.query(hv[:len(g["rs_ptr"]) - 1])) == _csr_lists(g, "rs")
        ts = (None, g["thresholds"].tolist()[0])
        _check_queries(ix, hv, qhv, ss, b, r, ts, alive)
        _check_pairs(ix, hv, ss, b, r, ts, alive)
        remap = np.asarray(ix.compact(), dtype=np.int64)
        assert np.array_equal(remap[alive], np.arange(alive.sum())) and np.all(remap[~alive] == -1)
        assert _lists(*ix.query(qhv)) == [sorted(int(remap[d]) for d in x) for x in _csr_lists(g, "rq")]
        _check_queries(ix, hv[alive], qhv, ss, b, r, ts)
        _check_pairs(ix, hv[alive], ss, b, r, ts)
    finally:
        ix.close()


# ---- constructed cases -------------------------------------------------------------------------------------------------
def test_samples_are_counted_not_words(be):
    """Document A agrees with the query on c samples and, elsewhere, on every k but no t; document B on every t but no k.
    A count of equal WORDS would give them ss + c; the sample count is c, so c / ss keeps both and (c + 1) / ss neither."""
    ss, b, r, c = 16, 4, 2, 6
    rs = np.random.RandomState(2)
    q = np.stack([rs.randint(0, 1 << 32, ss, dtype=np.uint64).astype(np.int64), rs.randint(-50, 50, ss)], axis=-1)
    a, bb = q.copy(), q.copy()
    a[c:, 1] += 1000                                             # same k, other t outside the first c samples
    bb[c:, 0] = (bb[c:, 0] + 12345) % (1 << 32)                  # same t, other k
    rows = np.stack([a, bb])
    ix = be.index(ss, b, r, 4)
    try:
        ix.insert(rows)
        for t, want in ((None, {0: c, 1: c}), (c / ss, {0: c, 1: c}), ((c + 1) / ss, {})):
            assert _got(*ix.query_jaccard(q[None], t)) == [want], t
        assert ix.query_best(q[None], (c + 1) / ss)[0].tolist() == [-1]
        ptr, idx, eq = ix.pairs(c / ss)
        assert idx.tolist() == [0] and eq.tolist() == [_eq(a, bb)]
        _check_queries(ix, rows, q[None], ss, b, r, (None, c / ss, (c + 1) / ss))
        _check_pairs(ix, rows, ss, b, r, (None, 0.0, c / ss, 1.0))
    finally:
        ix.close()


def test_range_limits(be):
    """k = 2^32 - 1, t = -1, -2^31 and 2^31 - 1 are accepted and kept apart (t = -1 is not k = 2^32 - 1's word in the
    other half).  t = 2^31, t = -2^31 - 1, k = -1 and k = 2^32 are rejected with ValueError naming the bound, and the
    index is unchanged afterwards."""
    ss, b, r = 8, 4, 2
    base = np.stack([np.arange(ss, dtype=np.int64) * 7, np.arange(ss, dtype=np.int64) - 3], axis=-1)
    rows = []
    for kk, tt in (((1 << 32) - 1, -1), (5, -(1 << 31)), (5, (1 << 31) - 1), (0, 0), (0xFFFFFFFF, 0xFFFFFFF)):
        x = base.copy()
        x[:, 0], x[0, 1] = kk, tt
        rows.append(x)
    rows = np.stack(rows)
    ix = be.index(ss, b, r, 10)
    try:
        ix.insert(rows)
        _check_queries(ix, rows, rows, ss, b, r, (None, 1.0))
        before = _got(*ix.query_jaccard(rows))
        for kk, tt, bound in ((0, 1 << 31, "t values"), (0, -(1 << 31) - 1, "t values"), (-1, 0, "k values"),
                              (1 << 32, 0, "k values")):
            bad = rows.copy()
            bad[2, 3] = (kk, tt)
            for call in (lambda: ix.insert(bad), lambda: ix.query_jaccard(bad), lambda: ix.insert_unique(bad)):
                with pytest.raises(ValueError, match=bound):
                    call()
            assert len(ix) == len(rows) and _got(*ix.query_jaccard(rows)) == before
    finally:
        ix.close()


@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_over_2r_words(be, head_collides):
    """Band tuples of 2r words that share a fingerprint without being equal (hash_model second preimages in bands 0, 31
    and 35), and the tuple whose fingerprint is the tables' empty key: members of a colliding tuple are no candidates."""
    ss, b, r = 120, 40, 3
    w = 2 * r
    rs = np.random.RandomState(13 + head_collides)
    base = rs.randint(0, 1 << 32, size=(60, 2 * ss), dtype=np.uint64).astype(np.uint32)
    same, other, queries = [], [], []
    for band in (0, 31, 35):
        sl = slice(band * w, (band + 1) * w)
        for d in rs.permutation(len(base))[:40]:
            t2 = hm.second_preimage(base[d, sl], band, rs)
            if t2 is None:
                continue
            s = base[rs.randint(0, len(base), 2)].copy()
            s[:, sl] = base[d, sl]
            x = base[rs.randint(0, len(base), 2)].copy()
            x[:, sl] = t2
            same.append(s)
            other.append(x)
            q = rs.randint(0, 1 << 32, size=(2, 2 * ss), dtype=np.uint64).astype(np.uint32)
            q[0, sl], q[1, sl] = base[d, sl], t2
            queries.append(q)
            break
        else:
            pytest.fail("no second preimage found for band %d" % band)
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, w, rs)
        if e is not None:
            em = base[rs.randint(0, len(base), 3)].copy()
            em[:, band * w:(band + 1) * w] = e
            same.append(em)
            break
    else:
        pytest.fail("no empty-key tuple found")
    parts = [base] + (same + other if head_collides else other + same)
    words = np.concatenate(parts)
    fp = hm.band_fp(np.concatenate(same[:3] + other), b, w)
    assert len(np.unique(fp)) < fp.size
    rows, qs = _unpack(words), _unpack(np.concatenate(queries + [same[-1][:1], base[:4]]))
    assert np.array_equal(_pack_cpu(rows, ss), words)
    ix = be.index(ss, b, r, len(rows))
    try:
        for row in rows:
            ix.insert(row[None])
        ref = _check_queries(ix, rows, qs, ss, b, r, (None, 0.02))
        want = _want(ref, rows, qs, None)
        for j in range(3):                                           # each query meets its own tuple's rows only
            assert len(want[2 * j]) >= 3 and len(want[2 * j + 1]) >= 2 and not set(want[2 * j]) & set(want[2 * j + 1])
        assert len(want[6]) >= 3                                     # the empty-key tuple's members
        _check_pairs(ix, rows, ss, b, r, (None, 0.5))
    finally:
        ix.close()


def test_sample_size_2048_empty_and_one_document(be):
    """ss = 2048 (4096-word rows: fewer warps per CTA); an empty index and a one-document index."""
    ss, b, r = 2048, 16, 4
    rs = np.random.RandomState(8)
    rows = np.stack([rs.randint(0, 3, size=(40, ss)), rs.randint(-2, 2, size=(40, ss))], axis=-1).astype(np.int64)
    rows[:, b * r:, 0] = rs.randint(0, 1 << 32, size=(40, ss - b * r), dtype=np.uint64).astype(np.int64)
    rows[10:20] = rows[0:10]
    rows[20:25, b * r:] = rows[0:5, b * r:]
    ix = be.index(ss, b, r, 40)
    try:
        ptr, idx, eq = ix.query_jaccard(rows[:2])                     # empty index
        assert ptr.tolist() == [0, 0, 0] and len(idx) == 0
        assert [x.tolist() for x in ix.query_best(rows[:1])] == [[-1], [-1]]
        ix.insert(rows)
        _check_queries(ix, rows, rows[:30], ss, b, r, (None, 0.5, 1.0))
        _check_pairs(ix, rows, ss, b, r, (None, 0.9))
    finally:
        ix.close()
    ix = be.index(4, 2, 2, 3)
    one = np.array([[[1, 0], [2, -1], [3, 5], [4, 0]]], dtype=np.int64)
    try:
        ix.insert(one)
        assert _got(*ix.query_jaccard(one, 1.0)) == [{0: 4}]
        assert [x.tolist() for x in ix.query_best(one)] == [[0], [4]]
        near = one.copy()
        near[0, 3, 1] = 1
        assert _got(*ix.query_jaccard(near)) == [{0: 3}] and _got(*ix.query_jaccard(near, 1.0)) == [{}]
        assert ix.pairs()[0].tolist() == [0, 0] and ix.clusters().tolist() == [0]
    finally:
        ix.close()


def test_c_abi_validation(emu_lib):
    """min_count counts samples: ss is accepted, ss + 1 (a word count would allow up to 2 ss) is refused; b * r > ss is
    refused; insert_tokens on a weighted handle and an unaligned batch for insert_unique are refused."""
    lib, ss = emu_lib, 8
    h = ctypes.c_void_p()
    assert lib.dsk_lsh_create_weighted(ss, 3, 3, 10, 0, ctypes.byref(h)) == DSK_ERR_INVALID   # b * r = 9 > 8
    assert lib.dsk_lsh_create_weighted(ss, 4, 2, 10, 0, ctypes.byref(h)) == DSK_OK
    buf = _aligned(np.zeros(512, dtype=np.int64))
    try:
        rows = _aligned(np.arange(3 * 2 * ss, dtype=np.uint32).reshape(3, 2 * ss) % 5)
        assert lib.dsk_lsh_insert(h, _p(rows), 3, None) == DSK_OK
        for mc in (ss + 1, 2 * ss, -1):
            assert lib.dsk_lsh_pairs_count(h, mc, _p(buf), None) == DSK_ERR_INVALID
            assert b"min_count must be in [0, sample_size=8]" in lib.dsk_last_error()
            assert lib.dsk_lsh_query_best(h, _p(rows), 1, mc, _p(buf), _p(buf), None) == DSK_ERR_INVALID
        assert lib.dsk_lsh_pairs_count(h, ss, _p(buf), None) == DSK_OK
        assert lib.dsk_lsh_query_best(h, _p(rows), 1, ss, _p(buf), _p(buf), None) == DSK_OK
        a, bb = np.zeros(ss, dtype=np.uint64), np.ones(ss, dtype=np.uint64)
        ph = ctypes.c_void_p()
        assert lib.dsk_perm_create(_p(a), _p(bb), ss, 0, ctypes.byref(ph)) == DSK_OK
        off = _aligned(np.array([0, 4], dtype=np.int64))
        tok = _aligned(np.arange(4, dtype=np.uint32))
        assert lib.dsk_lsh_insert_tokens(h, ph, _p(tok), 0, _p(off), 1, 4, None) == DSK_ERR_INVALID
        assert b"weighted" in lib.dsk_last_error()
        lib.dsk_perm_destroy(ph)
        ws_bytes = int(lib.dsk_lsh_unique_workspace_size(h, 2))
        ws = _aligned(np.zeros(ws_bytes, dtype=np.uint8))
        big = _aligned(np.zeros(2 * 2 * ss + 2, dtype=np.uint32))
        unal = ctypes.c_void_p(big.ctypes.data + 4)                  # 4-byte but not 8-byte aligned
        assert lib.dsk_lsh_unique_count(h, unal, 2, 0, _p(ws), ws_bytes, _p(buf), None) == DSK_ERR_ALIGN
        size = ctypes.c_int64()
        assert lib.dsk_lsh_size(h, ctypes.byref(size), None) == DSK_OK and size.value == 3
    finally:
        lib.dsk_lsh_destroy(h)


def test_packing_and_input_forms_cpu():
    """The packer: word 2j = k as uint32, word 2j + 1 = t as int32; a numpy array, a tensor and a list of WeightedMinHash
    give the same words; a 2-D MinHash matrix and a wrong sample size raise ValueError, floats TypeError."""
    import torch
    from datasketch_b200 import WeightedMinHash
    from datasketch_b200.lsh import _pack_weighted
    rows = np.array([[[0, 0], [(1 << 32) - 1, -1], [7, -(1 << 31)], [1 << 31, (1 << 31) - 1]]], dtype=np.int64)
    w = _pack_cpu(rows, 4)
    assert w.tolist() == [[0, 0, 0xFFFFFFFF, 0xFFFFFFFF, 7, 0x80000000, 0x80000000, 0x7FFFFFFF]]
    assert np.array_equal(_pack_cpu(torch.from_numpy(rows), 4), w)
    assert np.array_equal(_pack_cpu([WeightedMinHash(1, rows[0])], 4), w)
    assert np.array_equal(_pack_cpu(rows.astype(np.uint64)[:, :1], 1), w[:, :2])
    assert _pack_cpu([], 4).shape == (0, 8)
    with pytest.raises(ValueError, match="shape"):
        _pack_weighted(np.zeros((2, 8), dtype=np.uint32), 4, "cpu")
    with pytest.raises(ValueError, match="shape"):
        _pack_weighted(rows[:, :3], 4, "cpu")
    with pytest.raises(TypeError):
        _pack_weighted(rows.astype(np.float64), 4, "cpu")
    with pytest.raises(ValueError, match="t values"):
        _pack_weighted(np.array([[[0, (1 << 63) + 1]]], dtype=np.uint64), 1, "cpu")


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_api_errors():
    """A 2-D MinHash matrix or another sample size raises ValueError, insert_tokens raises on a weighted index, and the
    unweighted GpuLSH is unchanged by the new keyword."""
    import torch
    import datasketch_b200 as dsk
    ix = dsk.GpuLSH(num_perm=16, params=(4, 2), capacity=10, weighted=True)
    assert ix.weighted and (ix.b, ix.r, ix.h) == (4, 2, 16)
    for fn in (ix.insert, ix.query, ix.query_jaccard, ix.query_best, ix.insert_unique):
        with pytest.raises(ValueError):
            fn(np.zeros((2, 16), dtype=np.uint32))
        with pytest.raises(ValueError):
            fn(np.zeros((2, 8, 2), dtype=np.int64))
    tok = torch.zeros(4, dtype=torch.int32, device="cuda")
    off = torch.tensor([0, 4], dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="weighted"):
        ix.insert_tokens(tok, off, 4, np.ones((2, 16), dtype=np.uint64))
    assert len(ix) == 0
    plain = dsk.GpuLSH(num_perm=16, params=(4, 2), capacity=10)
    assert not plain.weighted
    plain.insert(np.arange(32, dtype=np.uint32).reshape(2, 16))
    assert len(plain) == 2


@pytest.mark.gpu
def test_reference_weighted_lsh_cases_replayed():
    """test/test_lsh.py's TestWeightedMinHashLSH (init, insert, query, remove) on GpuLSH(weighted=True) with the package's
    WeightedMinHashGenerator (sample size 4, dim 10)."""
    import datasketch_b200 as dsk
    lsh = dsk.GpuLSH(threshold=0.8, weighted=True)
    b1, r1 = lsh.b, lsh.r
    lsh = dsk.GpuLSH(threshold=0.8, weights=(0.2, 0.8), weighted=True)
    assert b1 < lsh.b and r1 > lsh.r
    rs = np.random.RandomState(0)
    mg = dsk.WeightedMinHashGenerator(10, 4)
    m1, m2 = mg.minhash(rs.uniform(1, 10, 10)), mg.minhash(rs.uniform(1, 10, 10))
    lsh = dsk.GpuLSH(threshold=0.5, num_perm=4, capacity=8, weighted=True)
    lsh.insert([m1, m2], keys=["a", "b"])
    assert "a" in lsh.query_keys([m1])[0] and "b" in lsh.query_keys([m2])[0]
    assert lsh.query_jaccard([m1])[2].max() == 4
    m3 = dsk.WeightedMinHashGenerator(10, 5).minhash(rs.uniform(1, 10, 10))
    with pytest.raises(ValueError):
        lsh.insert([m3])
    with pytest.raises(ValueError):
        lsh.query([m3])
    lsh.remove(0)
    assert 0 not in lsh.query([m1])[1].tolist() and 1 in lsh.query([m2])[1].tolist()
    with pytest.raises(ValueError):
        lsh.remove(0)


@pytest.mark.gpu
def test_device_pipeline_equals_the_host_path():
    """minhash_batch(to_host=False) gives the to_host rows as a CUDA int64 tensor, still refuses all-zero rows, and an
    index built from it answers exactly as one built from the host array."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(3)
    X = (rs.randint(1, 20, size=(3000, 96)) * (rs.rand(3000, 96) >= 0.6)).astype(np.float32)
    X[0] = 1.0
    X[1000:1500] = X[:500] * (rs.rand(500, 96) >= 0.1)
    X[X.sum(1) == 0, 0] = 1.0
    mg = dsk.WeightedMinHashGenerator(96, sample_size=64, seed=2)
    host = mg.minhash_batch(X)
    dev = mg.minhash_batch(X, to_host=False)
    assert dev.is_cuda and dev.dtype == torch.int64 and np.array_equal(dev.cpu().numpy(), host)
    with pytest.raises(ValueError, match="all zeros"):
        mg.minhash_batch(np.zeros((2, 96), dtype=np.float32), to_host=False)
    a = dsk.GpuLSH(threshold=0.7, num_perm=64, capacity=3000, weighted=True)
    b = dsk.GpuLSH(threshold=0.7, num_perm=64, capacity=3000, weighted=True)
    a.insert(dev)
    b.insert(host)
    pa, pb = a.candidate_pairs(0.7), b.candidate_pairs(0.7)   # CSR lists are in no particular order within a row
    assert np.array_equal(pa[0], pb[0]) and pa[0][-1] >= 300
    assert _got(*pa) == _got(*pb)
    assert _got(*a.query_jaccard(dev[:500], 0.5)) == _got(*b.query_jaccard(host[:500], 0.5))


@pytest.mark.gpu
def test_scale_one_million_vectors_100k_queries():
    """1M weighted signatures (ss = 64) with planted near-duplicates and 100k queries: query_jaccard and query_best equal
    a brute-force torch check on 300 sampled queries (every document sharing a band's 2r words, eq counted per sample)."""
    import torch
    import datasketch_b200 as dsk
    from datasketch_b200.lsh import _pack_weighted
    n, nq, ss, dim = 1_000_000, 100_000, 64, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    X = torch.randint(1, 20, (n, dim), device="cuda", generator=g).float()
    X *= torch.rand((n, dim), device="cuda", generator=g) >= 0.6
    src = torch.randint(0, n, (n // 10,), device="cuda", generator=g)
    X[: n // 10] = X[src] * (torch.rand((n // 10, dim), device="cuda", generator=g) >= 0.1)
    X[:, 0] += 1.0
    Q = X[torch.randint(0, n, (nq,), device="cuda", generator=g)].clone()
    Q *= torch.rand((nq, dim), device="cuda", generator=g) >= 0.15
    Q[:, 0] += 1.0
    mg = dsk.WeightedMinHashGenerator(dim, sample_size=ss, seed=1)
    sig = mg.minhash_batch(X, to_host=False)
    qsig = mg.minhash_batch(Q, to_host=False)
    ix = dsk.GpuLSH(threshold=0.8, num_perm=ss, capacity=n, weighted=True)
    ix.insert(sig)
    b, r = ix.b, ix.r
    ptr, idx, eq = ix.query_jaccard(qsig)
    bi, bq = ix.query_best(qsig, 0.8)
    assert ptr[-1] >= nq // 4
    words, qwords = _pack_weighted(sig, ss, 0), _pack_weighted(qsig, ss, 0)
    mc = _mc(0.8, ss)
    for q in np.random.RandomState(1).choice(nq, 300, replace=False).tolist():
        qw = qwords[q]
        band = (words[:, :2 * b * r].view(n, b, 2 * r) == qw[:2 * b * r].view(b, 2 * r)).all(-1).any(-1)
        cand = torch.nonzero(band).flatten()
        ceq = (words[cand].view(-1, ss, 2) == qw.view(ss, 2)).all(-1).sum(-1)
        want = dict(zip(cand.tolist(), ceq.tolist()))
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        assert dict(zip(idx[sl].tolist(), eq[sl].tolist())) == want, q
        kept = [(-e, d) for d, e in want.items() if e >= mc]
        e, d = min(kept) if kept else (1, -1)
        assert (int(bi[q]), int(bq[q])) == ((d, -e) if kept else (-1, -1)), q
