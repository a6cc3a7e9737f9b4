"""GpuLSHForest.query_topk / neighbors: each query's and each indexed document's forest candidates ranked by Jaccard
similarity on the device (forest_query_kernel's QUERY_TOPK and SELF_TOPK modes, DESIGN.md section 4j).

For a query m and a MinHashLSHForest holding the same documents in the same order, row q of ``query_topk(sig, k, c, t)``
is ``sorted([d for d in forest.query(m, c) if m.jaccard(doc[d]) >= t], key=lambda d: (-m.jaccard(doc[d]), d))[:k]``; a
``neighbors`` row ranks the first c distinct documents other than i of the same walk of document i's row.

CPU part: the C-ABI on the emulated library (2 SMs, 8 CTAs of 4 warps per SM: 64 queries per grid), with tree orders
from ``np.lexsort`` over the packed words, against tests/golden/forest_ranked.npz (the reference's own query, _query and
jaccard; oracle/gen_golden_forest_ranked.py) and against a numpy model over this package's host MinHashLSHForest.  GPU
part: the Python API, the fixture, and a 1M-document forest against query + codec.jaccard_pairs + a torch sort."""
import shutil

import numpy as np
import pytest

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
CONFIGS = ("w0", "w1", "w2", "w3", "u8", "u32")


@pytest.fixture(scope="module")
def dsk():
    import datasketch_b200
    return datasketch_b200


def cands(k):
    return sorted({k, 2 * k, 100})


def pack(hv):
    """[N, ss, 2] (k, t) integers -> [N, 2 * ss] uint32 words: k as uint32, t as int32 two's complement."""
    hv = np.asarray(hv, dtype=np.int64)
    return np.ascontiguousarray((hv & 0xFFFFFFFF).astype(np.uint32).reshape(len(hv), -1))


def orders(words, l, kw):
    """[l, n] tree orders: documents sorted by the tree's kw words (unsigned), then by number."""
    n = len(words)
    return np.ascontiguousarray(np.stack([np.lexsort([np.arange(n)] + [words[:, t * kw + c] for c in range(kw - 1, -1, -1)])
                                          for t in range(l)]).astype(np.int32).reshape(l, n))


class Forest:
    """A forest as the C-ABI sees it: packed rows, geometry and tree orders."""

    def __init__(self, words, num_perm, l, weighted):
        self.words = np.ascontiguousarray(words, dtype=np.uint32)
        self.num_perm, self.l, self.k, self.weighted = num_perm, l, num_perm // l, int(weighted)
        self.sw = 2 if weighted else 1
        self.n = len(words)
        self.order = orders(self.words, l, self.sw * self.k) if self.n else np.zeros((l, 0), np.int32)

    def _ptrs(self):
        return (self.words.ctypes.data, self.order.ctypes.data) if self.n else (None, None)

    def query(self, lib, q, topk):
        q = np.ascontiguousarray(q, dtype=np.uint32)
        out = np.full((len(q), topk), -7, dtype=np.int32)
        s, o = self._ptrs()
        fn = lib.dsk_forest_query_weighted if self.weighted else lib.dsk_forest_query
        assert fn(s, o, self.n, self.num_perm, self.l, self.k, q.ctypes.data if len(q) else None, len(q), topk,
                  out.ctypes.data, None) == 0
        return out

    def topk(self, lib, q, k, c, mc=0):
        q = np.ascontiguousarray(q, dtype=np.uint32)
        idx = np.full((len(q), k), -7, dtype=np.int32)
        eq = np.full((len(q), k), -7, dtype=np.int32)
        s, o = self._ptrs()
        rc = lib.dsk_forest_query_topk(s, o, self.n, self.num_perm, self.weighted, self.l, self.k,
                                       q.ctypes.data if len(q) else None, len(q), c, mc, k, idx.ctypes.data,
                                       eq.ctypes.data, None)
        assert rc == 0
        return idx, eq

    def neighbors(self, lib, k, c, mc=0):
        idx = np.full((self.n, k), -7, dtype=np.int32)
        eq = np.full((self.n, k), -7, dtype=np.int32)
        s, o = self._ptrs()
        assert lib.dsk_forest_neighbors(s, o, self.n, self.num_perm, self.weighted, self.l, self.k, c, mc, k,
                                        idx.ctypes.data, eq.ctypes.data, None) == 0
        return idx, eq


# ---- the numpy model: the walk in reference order, eq over all positions ---------------------------------------------
def _host(dsk, f):
    """This package's host MinHashLSHForest over the same rows (its query sets equal the reference's,
    tests/test_lshforest.py and tests/test_lshforest_weighted.py)."""
    h = dsk.MinHashLSHForest(num_perm=f.num_perm, l=f.l)
    for i in range(f.n):
        h.add(i, _obj(dsk, f, f.words[i]))
    h.index()
    return h


def _obj(dsk, f, row):
    if f.weighted:
        w = row.reshape(-1, 2)
        hv = np.stack([w[:, 0].astype(np.int64), w[:, 1].view(np.int32).astype(np.int64)], axis=1)
        return dsk.WeightedMinHash(1, hv)
    return dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64))


def eq_of(f, row, d):
    if f.weighted:
        return int((f.words[d].reshape(-1, 2) == row.reshape(-1, 2)).all(axis=1).sum())
    return int((f.words[d] == row).sum())


def walk(h, m, c, skip=None):
    res = set()
    for r in range(h.k, 0, -1):
        for d in h._query(m, r, h.l):
            if d != skip:
                res.add(d)
            if len(res) >= c:
                return res
    return res


def rank(f, row, cand, k, mc):
    kept = [(-eq_of(f, row, d), d) for d in cand]
    best = sorted(x for x in kept if -x[0] >= mc)[:k]
    idx = np.full(k, -1, np.int32)
    eq = np.full(k, -1, np.int32)
    idx[:len(best)] = [d for _, d in best]
    eq[:len(best)] = [-e for e, _ in best]
    return idx, eq


def model_topk(dsk, f, h, q, k, c, mc=0):
    rows = [rank(f, row, walk(h, _obj(dsk, f, row), c), k, mc) for row in q]
    return np.stack([x[0] for x in rows]).reshape(len(q), k), np.stack([x[1] for x in rows]).reshape(len(q), k)


def model_neighbors(dsk, f, h, k, c, mc=0, rows=None):
    rows = range(f.n) if rows is None else rows
    res = [rank(f, f.words[i], walk(h, _obj(dsk, f, f.words[i]), c, skip=i), k, mc) for i in rows]
    return np.stack([x[0] for x in res]), np.stack([x[1] for x in res])


def low_entropy(rs, n, K, dup=0, hi=3):
    """values 0..hi-1: long shared prefixes, large buckets at every r, many ties of eq"""
    sig = rs.randint(0, hi, size=(n, K)).astype(np.uint32)
    if dup:
        sig[rs.randint(0, n, dup)] = sig[rs.randint(0, n, dup)]
    return sig


def low_entropy_weighted(rs, n, ss, dup=0):
    """(k, t) samples with k in 0..2 and t in {-1, 0}: a negative t sorts after the others"""
    hv = np.stack([rs.randint(0, 3, size=(n, ss)), -rs.randint(0, 2, size=(n, ss))], axis=-1)
    if dup:
        hv[rs.randint(0, n, dup)] = hv[rs.randint(0, n, dup)]
    return pack(hv)


# ---- CPU: the fixture ---------------------------------------------------------------------------------------------
def fixture_forest(g, name):
    ss, l, weighted = (int(x) for x in g[name + "_params"])
    if weighted:
        return Forest(pack(g[name + "_hv"]), ss, l, True), pack(g[name + "_qhv"])
    sig = np.load(__file__.rsplit("/", 1)[0] + "/golden/lsh.npz")["sig"].astype(np.uint32)
    qsig = np.load(__file__.rsplit("/", 1)[0] + "/golden/lsh_topk.npz")["qsig"].astype(np.uint32)
    return Forest(sig, ss, l, False), qsig


@needs_gxx
@pytest.mark.parametrize("name", CONFIGS)
def test_emulated_fixture_ranked_lists(emu_lib, golden, dsk, name):
    g = golden("forest_ranked")
    f, q = fixture_forest(g, name)
    n_self = int(g["n_self"])
    h = _host(dsk, f)
    for k, c in ((1, 2), (5, 100), (32, 32)):         # (the GPU test below runs every (k, c) of the fixture)
        for j, t in enumerate((None, 0.5)):
                mc = dsk.lsh._jaccard_min_count(t, f.num_perm)
                tag = "%s_%%s_k%d_c%d_t%d_" % (name, k, c, j)
                idx, eq = f.topk(emu_lib, q, k, c, mc)
                assert np.array_equal(idx, g[tag % "q" + "idx"]), (k, c, t)
                assert np.array_equal(np.where(eq >= 0, eq / f.num_perm, -1.0), g[tag % "q" + "jac"]), (k, c, t)
                nidx, neq = f.neighbors(emu_lib, k, c, mc)
                assert np.array_equal(nidx[:n_self], g[tag % "s" + "idx"]), (k, c, t)
                assert np.array_equal(np.where(neq[:n_self] >= 0, neq[:n_self] / f.num_perm, -1.0), g[tag % "s" + "jac"])
                if k == 5 and c == 100:   # and the numpy model over the host class, every row
                    m_idx, m_eq = model_topk(dsk, f, h, q, k, c, mc)
                    assert np.array_equal(idx, m_idx) and np.array_equal(eq, m_eq), (k, c, t)
                    m_idx, m_eq = model_neighbors(dsk, f, h, k, c, mc)
                    assert np.array_equal(nidx, m_idx) and np.array_equal(neq, m_eq), (k, c, t)


# ---- CPU: without an oracle ------------------------------------------------------------------------------------------
def _set_ranked(f, q, sets, k):
    """query(sig, c)'s sets sorted by (-eq, d) and cut at k"""
    return [rank(f, row, [int(d) for d in s if d >= 0], k, 0) for row, s in zip(q, sets)]


@needs_gxx
@pytest.mark.parametrize("weighted", [False, True])
def test_emulated_topk_is_the_query_set_ranked(emu_lib, weighted):
    rs = np.random.RandomState(7 + weighted)
    K, l, n = 24, 4, 700
    words = low_entropy_weighted(rs, n, K, dup=60) if weighted else low_entropy(rs, n, K, dup=60)
    f = Forest(words, K, l, weighted)
    nq = 2 * 64 + 9                                    # two sweeps of the emulated grid and a tail
    q = np.concatenate([words[:nq - 30], (low_entropy_weighted(rs, 30, K) if weighted else low_entropy(rs, 30, K))])
    for k, c in ((1, 40), (7, 7), (32, 33), (5, 300)):
        sets = f.query(emu_lib, q, c)
        idx, eq = f.topk(emu_lib, q, k, c)
        want = _set_ranked(f, q, sets, k)
        assert np.array_equal(idx, np.stack([w[0] for w in want])), (k, c)
        assert np.array_equal(eq, np.stack([w[1] for w in want])), (k, c)
        if k == c:                                     # the whole collected set comes back
            assert [sorted(r[r >= 0].tolist()) for r in idx] == [sorted(s[s >= 0].tolist()) for s in sets]
        # min_count only removes documents from the collected set
        for mc in (K // 2,):
            fidx, feq = f.topk(emu_lib, q, k, c, mc)
            for j in range(nq):
                keep = [(d, e) for d, e in zip(*_full(f, q[j], sets[j])) if e >= mc][:k]
                assert fidx[j][:len(keep)].tolist() == [d for d, _ in keep] and (fidx[j][len(keep):] == -1).all()
                assert feq[j][:len(keep)].tolist() == [e for _, e in keep] and (feq[j][len(keep):] == -1).all()


def _full(f, row, s):
    idx, eq = rank(f, row, [int(d) for d in s if d >= 0], len(s), 0)
    keep = idx >= 0
    return idx[keep].tolist(), eq[keep].tolist()


@needs_gxx
@pytest.mark.parametrize("weighted", [False, True])
def test_emulated_neighbors_are_self_skipping_queries(emu_lib, dsk, weighted):
    """Row i == the ranking of the first c distinct documents other than i: query(row i, c + 1) without i when i is
    among them, else query(row i, c).  Exact copies of i (dup) stay neighbours."""
    rs = np.random.RandomState(11 + weighted)
    K, l, n = 16, 4, 300
    words = low_entropy_weighted(rs, n, K, dup=40) if weighted else low_entropy(rs, n, K, dup=40)
    f = Forest(words, K, l, weighted)
    h = _host(dsk, f)
    for k, c in ((1, 1), (32, 32), (10, 64), (4, 1024)):
        nidx, neq = f.neighbors(emu_lib, k, c)
        if c < 1024:
            s1, s0 = f.query(emu_lib, words, c + 1), f.query(emu_lib, words, c)
            for i in range(n):
                s = [d for d in s1[i] if d != i] if i in s1[i] else list(s0[i])
                want = rank(f, words[i], [int(d) for d in s if d >= 0], k, 0)
                assert np.array_equal(nidx[i], want[0]) and np.array_equal(neq[i], want[1]), (k, c, i)
        m_idx, m_eq = model_neighbors(dsk, f, h, k, c, rows=range(0, n, 7))
        assert np.array_equal(nidx[::7], m_idx) and np.array_equal(neq[::7], m_eq), (k, c)
        assert not (nidx == np.arange(n)[:, None]).any()


@needs_gxx
@pytest.mark.parametrize("weighted", [False, True])
def test_emulated_columns_past_l_times_k(emu_lib, weighted):
    """Columns past l*k are never walked: the collected sets stay, and eq changes by the changed positions."""
    rs = np.random.RandomState(13 + weighted)
    ss, l, n = 30, 4, 400                              # k = 7: 28 samples walked, 2 not
    words = low_entropy_weighted(rs, n, ss, dup=40) if weighted else low_entropy(rs, n, ss, dup=40)
    q = np.concatenate([words[:50], low_entropy_weighted(rs, 20, ss) if weighted else low_entropy(rs, 20, ss)])
    sw = 2 if weighted else 1
    w2, q2 = words.copy(), q.copy()
    w2[:, sw * 28:] = rs.randint(0, 1 << 32, size=(n, sw * 2), dtype=np.uint64).astype(np.uint32)
    q2[:, sw * 28:] = rs.randint(0, 1 << 32, size=(len(q), sw * 2), dtype=np.uint64).astype(np.uint32)
    f, f2 = Forest(words, ss, l, weighted), Forest(w2, ss, l, weighted)
    for c in (5, 40):
        a, b = f.query(emu_lib, q, c), f2.query(emu_lib, q2, c)
        assert [sorted(r) for r in a] == [sorted(r) for r in b]
        idx, eq = f2.topk(emu_lib, q2, min(c, 32), c)
        want = _set_ranked(f2, q2, b, min(c, 32))
        assert np.array_equal(idx, np.stack([x[0] for x in want])) and np.array_equal(eq, np.stack([x[1] for x in want]))
        idx1, eq1 = f.topk(emu_lib, q, min(c, 32), c)
        for j in range(len(q)):                        # per document, eq differs by the tail positions' agreement
            for d, e in zip(idx1[j], eq1[j]):
                if d >= 0:
                    head = eq_of(f, q[j], d) - _tail_eq(words[d], q[j], sw)
                    assert e == head + _tail_eq(words[d], q[j], sw)
                    assert eq_of(f2, q2[j], d) == head + _tail_eq(w2[d], q2[j], sw)


def _tail_eq(a, b, sw):
    a, b = a[sw * 28:].reshape(-1, sw), b[sw * 28:].reshape(-1, sw)
    return int((a == b).all(axis=1).sum())


@needs_gxx
def test_emulated_ties_and_large_buckets(emu_lib):
    """Every candidate of a bucket far larger than c at every r, eq taking few values: ties across lanes go to the
    smaller number, and the list cuts exactly where the reference's walk stops."""
    rs = np.random.RandomState(17)
    K, l, n = 8, 2, 1500
    words = low_entropy(rs, n, K, hi=2)
    f = Forest(words, K, l, False)
    q = np.concatenate([words[:40], low_entropy(rs, 30, K, hi=2)])
    for k, c in ((32, 1024), (32, 100), (8, 9)):
        sets = f.query(emu_lib, q, c)
        idx, eq = f.topk(emu_lib, q, k, c)
        want = _set_ranked(f, q, sets, k)
        assert np.array_equal(idx, np.stack([w[0] for w in want])) and np.array_equal(eq, np.stack([w[1] for w in want]))
        assert ((sets >= 0).sum(axis=1) == c).all()    # every walk stopped at c
        assert (np.diff(eq, axis=1) <= 0).all() and (eq[:, -1] >= 0).all()


@needs_gxx
@pytest.mark.parametrize("K,weighted", [(2048, False), (4096, False), (2048, True)])
def test_emulated_long_rows(emu_lib, K, weighted):
    """K = 2048 and 4096 words (the weighted case: 2048 samples = 4096 words)."""
    rs = np.random.RandomState(K + weighted)
    n, l = 48, 4
    if weighted:
        base = low_entropy_weighted(rs, 12, K)
    else:
        base = rs.randint(0, 1 << 32, size=(12, K), dtype=np.uint64).astype(np.uint32)
    words = base[rs.randint(0, 12, n)].copy()
    flip = rs.rand(*words.shape) < 0.3
    words[flip] = rs.randint(0, 4, size=int(flip.sum())).astype(np.uint32)
    f = Forest(words, K, l, weighted)
    q = words[:8].copy()
    for k, c in ((5, 10), (32, 40)):
        sets = f.query(emu_lib, q, c)
        idx, eq = f.topk(emu_lib, q, k, c)
        want = _set_ranked(f, q, sets, k)
        assert np.array_equal(idx, np.stack([w[0] for w in want])) and np.array_equal(eq, np.stack([w[1] for w in want]))
        nidx, neq = f.neighbors(emu_lib, k, c)
        assert not (nidx == np.arange(n)[:, None]).any()
        assert (neq[nidx >= 0] > 0).all()


@needs_gxx
@pytest.mark.parametrize("weighted", [False, True])
def test_emulated_empty_one_document_and_no_queries(emu_lib, weighted):
    K, l = 8, 2
    rs = np.random.RandomState(19)
    q = low_entropy_weighted(rs, 70, K) if weighted else low_entropy(rs, 70, K)
    empty = Forest(np.zeros((0, K * (2 if weighted else 1)), np.uint32), K, l, weighted)
    idx, eq = empty.topk(emu_lib, q, 5, 10)
    assert (idx == -1).all() and (eq == -1).all()
    assert empty.neighbors(emu_lib, 5, 10)[0].shape == (0, 5)
    one = Forest(q[:1], K, l, weighted)
    idx, eq = one.topk(emu_lib, q, 3, 3)
    hit = (q == q[0]).all(axis=1)
    assert (idx[hit, 0] == 0).all() and (eq[hit, 0] == K).all() and (idx[:, 1:] == -1).all()
    nidx, neq = one.neighbors(emu_lib, 3, 3)
    assert (nidx == -1).all() and (neq == -1).all()
    idx, eq = one.topk(emu_lib, q[:0], 3, 3)
    assert idx.shape == (0, 3)


@needs_gxx
def test_emulated_c_abi_errors(emu_lib):
    lib = emu_lib
    rs = np.random.RandomState(23)
    words = low_entropy(rs, 50, 16)
    f = Forest(words, 16, 4, False)
    q = words[:3].copy()
    out = np.zeros((50, 32), np.int32)                 # room for the neighbour rows of all 50 documents
    eq = np.zeros((50, 32), np.int32)
    s, o = f.words.ctypes.data, f.order.ctypes.data

    def topk(n=50, num_perm=16, weighted=0, l=4, k=4, qp=q.ctypes.data, nq=3, c=10, mc=0, kk=5, ip=out.ctypes.data,
             ep=eq.ctypes.data, sp=s):
        return lib.dsk_forest_query_topk(sp, o, n, num_perm, weighted, l, k, qp, nq, c, mc, kk, ip, ep, None)

    def nb(n=50, num_perm=16, weighted=0, l=4, k=4, c=10, mc=0, kk=5, ip=out.ctypes.data, sp=s):
        return lib.dsk_forest_neighbors(sp, o, n, num_perm, weighted, l, k, c, mc, kk, ip, eq.ctypes.data, None)

    assert topk() == 0 and nb() == 0
    for bad in (dict(l=5), dict(k=5), dict(kk=0), dict(kk=33), dict(c=4), dict(c=1025), dict(mc=-1), dict(mc=17),
                dict(weighted=2), dict(ip=None), dict(sp=None)):
        assert topk(**bad) != 0, bad
        assert "dsk_forest_query_topk" in lib.dsk_last_error().decode()
        if "qp" not in bad:
            assert nb(**bad) != 0, bad
    assert topk(qp=None) != 0
    assert topk(nq=0, qp=None, ip=None, ep=None) == 0           # no queries: no work, no buffers needed
    assert lib.dsk_forest_neighbors(None, None, 0, 16, 0, 4, 4, 10, 0, 5, None, None, None) == 0   # empty index
    # weighted rows must be 8-byte aligned
    wf = Forest(low_entropy_weighted(rs, 20, 8), 8, 2, True)
    raw = np.zeros(2 * 16 + 1, np.uint32)
    mis = raw[1:].view(np.uint32)
    assert lib.dsk_forest_query_topk(wf.words.ctypes.data, wf.order.ctypes.data, 20, 8, 1, 2, 4, mis.ctypes.data, 1, 5, 0,
                                     5, out.ctypes.data, eq.ctypes.data, None) != 0
    assert lib.dsk_forest_query_weighted(wf.words.ctypes.data, wf.order.ctypes.data, 20, 8, 2, 4, mis.ctypes.data, 1, 5,
                                         out.ctypes.data, None) != 0
    assert lib.dsk_forest_query_weighted(wf.words.ctypes.data, wf.order.ctypes.data, 20, 8, 2, 4, raw.ctypes.data, 1, 5,
                                         out.ctypes.data, None) == 0
    assert lib.dsk_forest_query_weighted(wf.words.ctypes.data, wf.order.ctypes.data, 20, 8, 3, 4, raw.ctypes.data, 1, 5,
                                         out.ctypes.data, None) != 0          # l * k > sample_size


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _dev(dsk, f):
    import torch
    dev = dsk.GpuLSHForest(num_perm=f.num_perm, l=f.l, weighted=bool(f.weighted))
    if f.weighted:
        w = f.words.reshape(f.n, -1, 2)
        dev.add(np.stack([w[..., 0].astype(np.int64), w[..., 1].view(np.int32).astype(np.int64)], axis=-1))
    else:
        dev.add(torch.from_numpy(f.words.view(np.int32)).cuda())
    dev.index()
    return dev


def _unpack(f, q):
    if not f.weighted:
        return q
    w = q.reshape(len(q), -1, 2)
    return np.stack([w[..., 0].astype(np.int64), w[..., 1].view(np.int32).astype(np.int64)], axis=-1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CONFIGS)
def test_fixture_through_the_class(golden, dsk, name):
    g = golden("forest_ranked")
    f, q = fixture_forest(g, name)
    n_self = int(g["n_self"])
    dev = _dev(dsk, f)
    qin = _unpack(f, q)
    for k in (1, 5, 32):
        for c in cands(k):
            for j, t in enumerate((None, 0.5)):
                tag = "%s_%%s_k%d_c%d_t%d_" % (name, k, c, j)
                idx, eq = dev.query_topk(qin, k, candidates=c, min_jaccard=t)
                assert np.array_equal(idx, g[tag % "q" + "idx"]), (k, c, t)
                assert np.array_equal(np.where(eq >= 0, eq / f.num_perm, -1.0), g[tag % "q" + "jac"])
                nidx, neq = dev.neighbors(k, candidates=c, min_jaccard=t)
                assert np.array_equal(nidx[:n_self], g[tag % "s" + "idx"]), (k, c, t)
                assert np.array_equal(np.where(neq[:n_self] >= 0, neq[:n_self] / f.num_perm, -1.0), g[tag % "s" + "jac"])
    idx, _ = dev.query_topk(qin, 4)                      # candidates default to 2k
    assert np.array_equal(idx, dev.query_topk(qin, 4, candidates=8)[0])


@pytest.mark.gpu
def test_python_errors_and_shapes(dsk):
    rs = np.random.RandomState(29)
    sig = low_entropy(rs, 200, 32, dup=20)
    dev = dsk.GpuLSHForest(num_perm=32, l=4)
    dev.add(sig)
    with pytest.raises(ValueError):
        dev.query_topk(sig[:3], 5)                     # index() has not been called
    with pytest.raises(ValueError):
        dev.neighbors(5)
    dev.index()
    for bad in (0, 33, 2.0, True, None):
        with pytest.raises(ValueError):
            dev.query_topk(sig[:3], bad)
        with pytest.raises(ValueError):
            dev.neighbors(bad)
    for bad in (4, 1025, 10.0, True):
        with pytest.raises(ValueError):
            dev.query_topk(sig[:3], 5, candidates=bad)
        with pytest.raises(ValueError):
            dev.neighbors(5, candidates=bad)
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            dev.query_topk(sig[:3], 5, min_jaccard=bad)
    idx, eq = dev.query_topk(sig[:0], 5)
    assert idx.shape == (0, 5) and eq.shape == (0, 5)
    idx, eq = dev.query_topk(sig[:10], 5, candidates=1024, to_host=False)
    assert idx.is_cuda and idx.shape == (10, 5)
    empty = dsk.GpuLSHForest(num_perm=32, l=4)
    empty.index()
    idx, eq = empty.query_topk(sig[:7], 3)
    assert (idx == -1).all() and (eq == -1).all()
    assert empty.neighbors(3)[0].shape == (0, 3)


def _planted(rs, n, K, groups):
    """n random rows with near-duplicate groups: each group row copies a base and re-draws a share of positions"""
    sig = rs.randint(0, 1 << 32, size=(n, K), dtype=np.uint64).astype(np.uint32)
    base = rs.randint(0, n, groups)
    for frac in (0.05, 0.15, 0.3):
        tgt = rs.randint(0, n, groups)
        sig[tgt] = sig[base]
        m = rs.rand(groups, K) < frac
        sig[tgt] = np.where(m, rs.randint(0, 1 << 32, size=(groups, K), dtype=np.uint64).astype(np.uint32), sig[tgt])
    return sig


def flow_topk(dsk, dev, d_q, k, c):
    """The flow query_topk replaces: query(sig, c), codec.jaccard_pairs of every (query, document) pair, a torch sort."""
    import torch
    cand = dev.query(d_q, c, to_host=False).to(torch.int64)
    nq = cand.shape[0]
    both = torch.cat([dev._sig, d_q])                  # query q is row n + q
    qi = (torch.arange(nq, device=cand.device) + dev._sig.shape[0])[:, None].expand(nq, c)
    valid = cand >= 0
    jac = torch.from_numpy(dsk.codec.jaccard_pairs(both, qi[valid], cand[valid])).to(cand.device)
    eq = torch.full(cand.shape, -1, dtype=torch.int64, device=cand.device)
    eq[valid] = torch.round(jac * dev.h).to(torch.int64)
    key = torch.where(valid, -eq * (1 << 32) + cand, torch.full_like(cand, 1 << 62))
    o = torch.sort(key, dim=1).indices[:, :k]
    return torch.gather(cand, 1, o).to(torch.int32), torch.gather(eq, 1, o).to(torch.int32)


@pytest.mark.gpu
def test_million_signature_forest(dsk):
    import torch
    rs = np.random.RandomState(31)
    n, K, l, nq = 1_000_000, 128, 8, 100_000
    sig = _planted(rs, n, K, 100_000)
    d_sig = torch.from_numpy(sig.view(np.int32)).cuda()
    dev = dsk.GpuLSHForest(num_perm=K, l=l)
    dev.add(d_sig)
    dev.index()
    q = sig[rs.randint(0, n, nq)].copy()
    flip = rs.rand(nq, K) < 0.1
    q[flip] = rs.randint(0, 1 << 32, size=int(flip.sum()), dtype=np.uint64).astype(np.uint32)
    d_q = torch.from_numpy(q.view(np.int32)).cuda()
    for k, c in ((10, 20), (10, 100)):
        idx, eq = dev.query_topk(d_q, k, candidates=c, to_host=False)
        w_idx, w_eq = flow_topk(dsk, dev, d_q, k, c)
        assert torch.equal(idx, w_idx) and torch.equal(eq, w_eq), (k, c)
    nidx, neq = dev.neighbors(10)
    rows = rs.choice(n, 300, replace=False)
    f = Forest(sig, K, l, False)
    f.order = dev._order.cpu().numpy()
    for i in rows:   # the first 20 distinct documents other than i: query(row i, 21) without i, else query(row i, 20)
        s1 = dev.query(sig[i:i + 1], 21)[0]
        s = [int(d) for d in s1 if d >= 0 and d != i] if i in s1 else \
            [int(d) for d in dev.query(sig[i:i + 1], 20)[0] if d >= 0]
        want = rank(f, sig[i], s, 10, 0)
        assert np.array_equal(nidx[i], want[0]) and np.array_equal(neq[i], want[1]), i
