"""GpuLSH.query_topk / neighbors: each row's k most similar candidates, ranked on the device.

``query_topk(sig, k, min_jaccard)`` gives, per query row, the first k candidates of ``query_jaccard(sig, min_jaccard)`` in
the order larger eq first, then smaller document number, padded with -1 / -1: for a query m, ``sorted([d for d in
lsh.query(m) if m.jaccard(doc[d]) >= t], key=lambda d: (-m.jaccard(doc[d]), d))[:k]`` (lsh.py:370-432, minhash.py:324).
``neighbors(k, min_jaccard)`` gives the same list for every indexed document's own row, without the document itself;
a removed document's row is all -1.  The order is total, so both results are compared as arrays.

The oracle is oracle_np.DictLSH.query (with test_lsh_remove.py's MinHashLSH.remove) and oracle_np.jaccard (or
wmh_jaccard), sorted by (-eq, d) and cut at k; tests/golden/lsh_topk.npz (oracle/gen_golden_lsh_topk.py) pins it to the
reference.  The two backends are those of test_lsh_query_jaccard.py: ``emu``, the whole library on the emulation shim
driven through its C-ABI, and ``gpu``, the Python API on the H100.
"""
import os
import sys

import numpy as np
import pytest

from oracle import oracle_clib as oc
from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402
from test_lsh_self_join import _aligned, _low_entropy, _min_count, _p  # noqa: E402
from test_lsh_remove import _oracle_index  # noqa: E402
from test_lsh_query_jaccard import _EmuQIndex, _GpuQIndex, _got, _perturb, _want  # noqa: E402
from test_lsh_weighted import _EmuW, _GpuW, _golden as _wgolden, _mc, _oracle as _woracle, _want as _wwant  # noqa: E402

DSK_OK, DSK_ERR_INVALID = 0, 1


# ---- backends ----------------------------------------------------------------------------------------------------------
class _TopkC:
    """dsk_lsh_query_topk / dsk_lsh_neighbors through the C-ABI of the emulated library."""

    def query_topk(self, sig, k, t=None):
        lib, q, mc = self.lib, self._q(sig), self._m(t)
        nq = len(q)
        idx, eq = np.full((max(nq, 1), k), -7, dtype=np.int32), np.full((max(nq, 1), k), -7, dtype=np.int32)
        assert lib.dsk_lsh_query_topk(self.h, _p(q), nq, mc, k, _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return idx[:nq], eq[:nq]

    def neighbors(self, k, t=None):
        lib, n, mc = self.lib, self._size(), self._m(t)
        idx, eq = np.full((max(n, 1), k), -7, dtype=np.int32), np.full((max(n, 1), k), -7, dtype=np.int32)
        assert lib.dsk_lsh_neighbors(self.h, mc, k, _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return idx[:n], eq[:n]


class _EmuTIndex(_TopkC, _EmuQIndex):
    def _q(self, sig):
        return _aligned(np.asarray(sig, dtype=np.uint32))

    def _m(self, t):
        return _min_count(t, self.k)

    def _size(self):
        return self.n


class _EmuWTIndex(_TopkC, _EmuW):
    def _q(self, rows):
        return self._rows(rows)

    def _m(self, t):
        return _mc(t, self.ss)

    def _size(self):
        return len(self)


class _GpuTIndex(_GpuQIndex):
    def query_topk(self, sig, k, t=None):
        return self.ix.query_topk(np.ascontiguousarray(sig, dtype=np.uint32), k, t)

    def neighbors(self, k, t=None):
        return self.ix.neighbors(k, t)


class _Emu:
    name = "emu"
    grid_rows = 2 * 8 * 8          # two emulated SMs x 8 CTAs x 8 warps: rows one sweep of the walk covers

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuTIndex(self.lib, k, b, r, capacity)

    def windex(self, ss, b, r, capacity):
        return _EmuWTIndex(self.lib, ss, b, r, capacity)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk
        self.grid_rows = dsk._native.device_info(0)["sm_count"] * 8 * 8

    def index(self, k, b, r, capacity):
        return _GpuTIndex(self.dsk, k, b, r, capacity)

    def windex(self, ss, b, r, capacity):
        return _GpuW(self.dsk, ss, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
def _topk(dicts, k):
    """Per row {d: eq} -> (idx int32[R, k], eq int32[R, k]): sorted by (-eq, d), cut at k, padded with -1 / -1."""
    idx, eq = np.full((len(dicts), k), -1, dtype=np.int32), np.full((len(dicts), k), -1, dtype=np.int32)
    for q, w in enumerate(dicts):
        best = sorted(w.items(), key=lambda x: (-x[1], x[0]))[:k]
        idx[q, :len(best)] = [d for d, _ in best]
        eq[q, :len(best)] = [e for _, e in best]
    return idx, eq


def _nbr_dicts(ref, rows, t, alive, want=_want):
    """Per document i: {d: eq} over query(row i) without i (empty for a removed i)."""
    out = want(ref, rows, rows, t)
    for i, w in enumerate(out):
        w.pop(i, None)
        if not alive[i]:
            w.clear()
    return out


def _same(got, want, what):
    gi, ge = (np.asarray(x) for x in got)
    wi, we = want
    assert gi.shape == wi.shape and ge.shape == we.shape, what
    assert np.array_equal(gi, wi) and np.array_equal(ge, we), what


def _check(ix, rows, qsig, k, b, r, thresholds, ks=(1, 5, 32), alive=None):
    """query_topk of qsig and neighbors of the index against the oracle over rows (removed ones excluded)."""
    rows = np.asarray(rows, dtype=np.uint32)
    alive = np.ones(len(rows), dtype=bool) if alive is None else alive
    ref = _oracle_index(rows, alive, k, b, r)
    for t in thresholds:
        wq = _want(ref, rows, qsig, t)
        wn = _nbr_dicts(ref, rows, t, alive)
        for kk in ks:
            _same(ix.query_topk(qsig, kk, t), _topk(wq, kk), ("query_topk", kk, t))
            _same(ix.neighbors(kk, t), _topk(wn, kk), ("neighbors", kk, t))
    return ref


def _check_consistency(ix, rows, qsig, thresholds, ks=(1, 5, 32)):
    """Without the oracle: query_topk(sig, 1) == query_best; query_topk == sorted and cut query_jaccard; neighbors ==
    sorted and cut symmetrised candidate_pairs; neighbors row i == query_topk(own row i, k + 1) without i, cut at k."""
    n = len(rows)
    for t in thresholds:
        qj = _got(*ix.query_jaccard(qsig, t))
        ptr, idx, eq = ix.pairs(t)
        sym = [dict() for _ in range(n)]
        for i, d, e in zip(np.repeat(np.arange(n), np.diff(ptr)).tolist(), idx.tolist(), eq.tolist()):
            sym[i][d] = sym[d][i] = e
        bi, bq = ix.query_best(qsig, t)
        ti, tq = ix.query_topk(qsig, 1, t)
        assert np.array_equal(ti[:, 0], bi) and np.array_equal(tq[:, 0], bq), t
        for kk in ks:
            _same(ix.query_topk(qsig, kk, t), _topk(qj, kk), ("query_topk vs query_jaccard", kk, t))
            ni, ne = ix.neighbors(kk, t)
            _same((ni, ne), _topk(sym, kk), ("neighbors vs candidate_pairs", kk, t))
            if kk < 32:
                si, se = ix.query_topk(rows, kk + 1, t)
                for i in range(n):
                    keep = si[i] != i
                    assert np.array_equal(si[i][keep][:kk], ni[i]) and np.array_equal(se[i][keep][:kk], ne[i]), (i, kk, t)


# ---- order and ties ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,b,r,vals", [(32, 8, 4, 3), (100, 33, 3, 4)])
def test_low_entropy_big_buckets(be, k, b, r, vals):
    """Big buckets with many eq ties and (b = 33) two lane rounds; queries mix indexed rows, perturbed rows and unrelated
    rows.  Thresholds: none, 1.0 and the exact boundaries c / K and (c + 1) / K; k = 1, 5 and 32."""
    rs = np.random.RandomState(k + b + 1)
    n = (120 if b <= 32 else 80) if be.name == "emu" else 1500
    nq = 45 if be.name == "emu" else 900
    sig = _low_entropy(rs, n, k, vals)
    third = nq // 3
    qsig = np.concatenate([sig[rs.choice(n, third)], _perturb(rs, sig[rs.choice(n, third)], 0.1, vals),
                           _low_entropy(rs, nq - 2 * third, k, vals)])
    ix = be.index(k, b, r, n)
    ix.insert(sig[:n // 2])
    ix.insert(sig[n // 2:])
    try:
        c = k // 3
        _check(ix, sig, qsig, k, b, r, (None, 1.0, c / k, (c + 1) / k))
        _check_consistency(ix, sig, qsig, (None, c / k))
    finally:
        ix.close()


def test_ties_across_lanes_and_within_a_chain(be):
    """Twelve documents share the top eq with a query, two per band (one lane's chain, walked from the last inserted) over
    six bands (six lanes), in shuffled numbers; one is worse.  k = 5 keeps the five smallest tied numbers, k = 12 all
    ties, k = 13 the worse one last, k = 32 pads.  A unique better document inserted last comes first."""
    k, b, r = 64, 16, 4
    rs = np.random.RandomState(78)
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
    docs = []
    for j in range(6):                                           # eq = K - 8: bands 0..j-1 broken, band j intact
        for _ in range(2):
            d = q.copy()
            pos = [jj * r for jj in range(j)] + [(b - 1 - m) * r + 1 for m in range(8 - j)]
            d[pos] = d[pos] + 1 + rs.randint(0, 1000, size=len(pos)).astype(np.uint32)
            docs.append(d)
    worse = q.copy()                                             # eq = K - 9, met through band 0
    worse[[r + 1, 2 * r, 3 * r + 2, 5 * r, 6 * r, 7 * r + 3, 9 * r, 10 * r, 11 * r]] += 1
    docs.append(worse)
    noise = rs.randint(0, 1 << 32, size=(5, k), dtype=np.uint64).astype(np.uint32)
    rows = np.concatenate([noise, np.stack(docs)])
    order = rs.permutation(len(rows))
    rows = rows[order]
    ties = sorted(i for i in range(len(rows)) if len(noise) <= order[i] < len(noise) + 12)
    w = int(np.flatnonzero(order == len(noise) + 12)[0])
    ix = be.index(k, b, r, len(rows) + 1)
    try:
        for row in rows:
            ix.insert(row[None])
        for kk, want in ((1, ties[:1]), (5, ties[:5]), (12, ties), (13, ties + [w]), (32, ties + [w])):
            idx, eq = ix.query_topk(q[None], kk)
            assert idx[0].tolist() == want + [-1] * (kk - len(want)), kk
            assert eq[0].tolist() == [k - 8] * min(kk, 12) + [k - 9] * (len(want) - 12 if kk > 12 else 0) + \
                [-1] * (kk - len(want)), kk
        assert ix.query_topk(q[None], 32, (k - 8) / k)[0][0].tolist() == ties + [-1] * 20
        _check(ix, rows, np.stack([q, q ^ 1]), k, b, r, (None, (k - 8) / k), ks=(1, 3, 12, 13, 32))
        _check_consistency(ix, rows, np.stack([q]), (None,), ks=(1, 3, 13))
        better = q.copy()
        better[b * r - 1] += 1                                   # eq = K - 1, the largest number
        ix.insert(better[None])
        idx, eq = ix.query_topk(q[None], 3)
        assert idx[0].tolist() == [len(rows)] + ties[:2] and eq[0].tolist() == [k - 1, k - 8, k - 8]
    finally:
        ix.close()


def test_exactly_fewer_and_more_than_k_candidates(be):
    """A bucket of exactly k members, one of fewer and one of more: every slot filled, pads behind the fewer, the first k
    (by eq, then number) of the more -- for k = 1, 7 and 32.  Also the entry at position k - 1 of a full list."""
    k, b, r = 64, 8, 8
    rs = np.random.RandomState(12)
    groups = []
    for size in (7, 3, 40, 32, 31, 33):
        head = rs.randint(0, 1 << 32, size=r, dtype=np.uint64).astype(np.uint32)
        g = rs.randint(0, 1 << 32, size=(size, k), dtype=np.uint64).astype(np.uint32)
        g[:, :r] = head
        g[:, r:r + 20] = rs.randint(0, 1 << 32, size=20, dtype=np.uint64).astype(np.uint32)
        g[np.arange(size), r + (np.arange(size) % 20)] += 1        # eq = 27 or 28 with the group's first member's row
        groups.append(g)
    rows = np.concatenate(groups)
    rows = rows[rs.permutation(len(rows))]
    qsig = np.concatenate([g[:1] for g in groups])
    ix = be.index(k, b, r, len(rows))
    try:
        ix.insert(rows)
        _check(ix, rows, qsig, k, b, r, (None, 0.4), ks=(1, 3, 7, 31, 32))
        full = ix.query_topk(qsig, 32)[0]
        assert (full[2] >= 0).all() and (full[3] >= 0).all() and (full[4] >= 0).sum() == 31 and (full[1] >= 0).sum() == 3
        assert (ix.query_topk(qsig, 7)[0][0] >= 0).all() and (ix.query_topk(qsig, 7)[0][1] >= 0).sum() == 3
    finally:
        ix.close()


# ---- hash edge cases, removal, index variants --------------------------------------------------------------------------
@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_and_the_empty_key(be, head_collides):
    """Indexed tuples that share a band's fingerprint without being equal (hash_model second preimages in bands 0, 31 and
    35, the second lane round) and the tuple whose fingerprint is the tables' empty key, also at a chain's head: members of
    a colliding tuple are never listed, by query_topk or neighbors."""
    k, b, r = 120, 40, 3
    rs = np.random.RandomState(61 + head_collides)
    base = rs.randint(0, 1 << 32, size=(60, k), dtype=np.uint64).astype(np.uint32)
    same, other, queries = [], [], []
    for band in (0, 31, 35):
        sl = slice(band * r, (band + 1) * r)
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
            q = rs.randint(0, 1 << 32, size=(2, k), dtype=np.uint64).astype(np.uint32)
            q[0, sl], q[1, sl] = base[d, sl], t2
            queries.append(q)
            break
        else:
            pytest.fail("no second preimage found for band %d" % band)
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, r, rs)
        if e is not None:
            em = base[rs.randint(0, len(base), 3)].copy()
            em[:, band * r:(band + 1) * r] = e
            same.append(em)
            q = rs.randint(0, 1 << 32, size=(1, k), dtype=np.uint64).astype(np.uint32)
            q[0, band * r:(band + 1) * r] = e
            queries.append(q)
            break
    else:
        pytest.fail("no empty-key tuple found")
    parts = [base] + (same + other if head_collides else other + same)
    rows = np.concatenate(parts)
    qsig = np.concatenate(queries + [base[:5]])
    fp = hm.band_fp(np.concatenate(same[:3] + other), b, r)
    assert len(np.unique(fp)) < fp.size
    ix = be.index(k, b, r, len(rows))
    try:
        for p in parts:
            for row in p:                                            # one at a time: a known chain order
                ix.insert(row[None])
        ref = _check(ix, rows, qsig, k, b, r, (None, 0.05), ks=(1, 2, 32))
        want = _want(ref, rows, qsig, None)
        for j in range(3):                                           # each query meets its own tuple's rows only
            assert len(want[2 * j]) >= 3 and len(want[2 * j + 1]) >= 2 and not set(want[2 * j]) & set(want[2 * j + 1])
        assert len(want[6]) >= 3                                     # the empty-key tuple's members
    finally:
        ix.close()


def test_removed_documents_before_and_after_compact(be):
    """Removed chain heads, middles and tails (and a whole group): never listed, and their own neighbour rows are -1;
    after compact() rows and numbers follow remap."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(4)
    groups, size = 4, 6
    rows = rs.randint(0, 1 << 32, size=(groups * size + 10, k), dtype=np.uint64).astype(np.uint32)
    for g in range(groups):                                      # member j of group g is row j * groups + g
        rows[g:groups * size:groups, 0:r] = rs.randint(0, 1 << 32, size=r, dtype=np.uint64).astype(np.uint32)
        rows[g:groups * size:groups, r * 3:r * 4] = 17 + g
    qsig = np.concatenate([rows, _perturb(rs, rows, 0.2, 1 << 30)])
    qsig[len(rows):, 0:r] = rows[:, 0:r]
    ix = be.index(k, b, r, len(rows))
    try:
        for row in rows:
            ix.insert(row[None])
        alive = np.ones(len(rows), dtype=bool)
        for part in ([(size - 1) * groups + 0], [2 * groups + 1], [0 * groups + 2], list(range(3, groups * size, groups))):
            ix.remove(part)
            alive[part] = False
        thresholds = (None, 0.5)
        _check(ix, rows, qsig, k, b, r, thresholds, ks=(1, 3, 32), alive=alive)
        ni, ne = ix.neighbors(4)
        assert (ni[~alive] == -1).all() and (ne[~alive] == -1).all() and not np.isin(ni, np.flatnonzero(~alive)).any()
        before = {(t, kk): (ix.query_topk(qsig, kk, t), ix.neighbors(kk, t)) for t in thresholds for kk in (3, 32)}
        remap = np.asarray(ix.compact(), dtype=np.int64)
        _check(ix, rows[alive], qsig, k, b, r, thresholds, ks=(1, 3, 32))
        for (t, kk), ((qi, qe), (bi, bq)) in before.items():
            mapped = np.where(qi >= 0, remap[qi], -1)
            _same(ix.query_topk(qsig, kk, t), (mapped, qe), ("query_topk after compact", kk, t))
            _same(ix.neighbors(kk, t), (np.where(bi >= 0, remap[bi], -1)[alive], bq[alive]), ("neighbors", kk, t))
    finally:
        ix.close()


def test_rows_from_the_fused_token_insert(be):
    """Documents inserted from tokens (the signature kernel's fused insert epilogue) between plain inserts; near-duplicate
    queries of them, and neighbors of the whole index."""
    k, b, r = 128, 32, 4
    rs = np.random.RandomState(6)
    n = 90 if be.name == "emu" else 3000
    lens = rs.randint(1, 200, size=n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    perms = o.init_permutations(k, 5)
    sig = oc.minhash_bulk_u32tok(tok, off, perms)
    qtok = tok.copy()
    qtok[rs.rand(len(qtok)) < 0.1] = rs.randint(0, 1 << 32, dtype=np.uint64)
    qsig = oc.minhash_bulk_u32tok(qtok, off, perms)[:40]
    before = rs.randint(0, 1 << 32, size=(20, k), dtype=np.uint64).astype(np.uint32)
    ix = be.index(k, b, r, n + 40)
    try:
        ix.insert(before)
        ix.insert_tokens(tok, off, perms)
        ix.insert(sig[:20])
        rows = np.concatenate([before, sig, sig[:20]])
        ref = _check(ix, rows, qsig, k, b, r, (None, 0.7), ks=(1, 4, 32))
        assert sum(len(w) for w in _want(ref, rows, qsig, 0.7)) >= len(qsig) // 4
    finally:
        ix.close()


@pytest.mark.parametrize("cfg", ("a", "b", "c"))
def test_weighted_index(be, golden, cfg):
    """A weighted index (eq counts samples, SW = 2) over lsh_weighted.npz's three configurations: query_topk of the
    held-out rows and neighbors against the oracle (DictLSH over [ss, 2] rows, WeightedMinHash.jaccard)."""
    g = _wgolden(golden, cfg)
    b, r, ss = g["params"].tolist()
    hv, qhv = g["hv"], g["qhv"]
    alive = np.ones(len(hv), dtype=bool)
    ix = be.windex(ss, b, r, len(hv))
    try:
        ix.insert(hv)
        ref = _woracle(hv, alive, ss, b, r)
        for t in (None,) + tuple(g["thresholds"].tolist()):
            wq = _wwant(ref, hv, qhv, t)
            wn = _nbr_dicts(ref, hv, t, alive, want=_wwant)
            for kk in (1, 5, 32):
                _same(ix.query_topk(qhv, kk, t), _topk(wq, kk), ("query_topk", kk, t))
                _same(ix.neighbors(kk, t), _topk(wn, kk), ("neighbors", kk, t))
            bi, bq = ix.query_best(qhv, t)
            ti, tq = ix.query_topk(qhv, 1, t)
            assert np.array_equal(ti[:, 0], bi) and np.array_equal(tq[:, 0], bq)
        ix.remove(np.arange(0, len(hv), 3))
        alive[::3] = False
        ref = _woracle(hv, alive, ss, b, r)
        _same(ix.neighbors(8), _topk(_nbr_dicts(ref, hv, None, alive, want=_wwant), 8), "neighbors after remove")
        _same(ix.query_topk(qhv, 8), _topk(_wwant(ref, hv, qhv, None), 8), "query_topk after remove")
    finally:
        ix.close()


@pytest.mark.parametrize("k", [2048, 4096])
def test_large_k_fewer_warps_per_cta(be, k):
    """K = 2048 (4 warps per CTA) and K = 4096 (2 warps): each warp's row still fits the shared memory it is given."""
    b, r = 16, 4
    rs = np.random.RandomState(k + 1)
    n = 40
    sig = rs.randint(0, 4, size=(n, k)).astype(np.uint32)
    sig[:, b * r:] = rs.randint(0, 1 << 32, size=(n, k - b * r), dtype=np.uint64).astype(np.uint32)
    sig[10:20] = sig[0:10]
    sig[20:25, b * r:] = sig[0:5, b * r:]
    qsig = np.concatenate([sig[:12], _perturb(rs, sig[12:30], 0.3, 4)])
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        _check(ix, sig, qsig, k, b, r, (None, 0.5), ks=(1, 6, 32))
    finally:
        ix.close()


def test_more_rows_than_one_grid_sweep(be):
    """Queries and documents beyond one sweep of the grid: the walk's grid-stride loop over rows, in both modes."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(10)
    n = (2 if be.name == "emu" else 1) * be.grid_rows + 7
    sig = rs.randint(0, 1 << 32, size=(n, k), dtype=np.uint64).astype(np.uint32)
    sig[n // 2:] = _perturb(rs, sig[rs.randint(0, n // 2, n - n // 2)], 0.15, 1 << 30)   # near-copies of the first half
    nq = (3 if be.name == "emu" else 1) * be.grid_rows + 5
    qsig = _perturb(rs, sig[rs.randint(0, n, nq)], 0.1, 1 << 30)
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        _check(ix, sig, qsig, k, b, r, (None, 0.6), ks=(3, 32))
    finally:
        ix.close()


def test_empty_one_document_and_no_queries(be):
    k, b, r = 64, 8, 8
    ix = be.index(k, b, r, 10)
    row = np.arange(k, dtype=np.uint32)[None]
    try:
        for kk in (1, 32):                                          # empty index
            assert [x.tolist() for x in ix.query_topk(np.concatenate([row, row]), kk)] == [[[-1] * kk] * 2] * 2
            assert [x.shape for x in ix.neighbors(kk)] == [(0, kk), (0, kk)]
        ix.insert(row)
        for t in (None, 0.0, 1.0):
            assert [x.tolist() for x in ix.query_topk(row, 3, t)] == [[[0, -1, -1]], [[k, -1, -1]]]
            assert [x.tolist() for x in ix.neighbors(2, t)] == [[[-1, -1]], [[-1, -1]]]   # one document: no neighbour
        near = row.copy()
        near[0, 0] += 1
        assert [x.tolist() for x in ix.query_topk(near, 1, 1.0)] == [[[-1]], [[-1]]]
        assert [x.shape for x in ix.query_topk(np.zeros((0, k), dtype=np.uint32), 5)] == [(0, 5), (0, 5)]
        ix.insert(row)                                             # an exact copy: each is the other's neighbour
        assert [x.tolist() for x in ix.neighbors(2)] == [[[1, -1], [0, -1]], [[k, -1], [k, -1]]]
    finally:
        ix.close()


# ---- errors ------------------------------------------------------------------------------------------------------------
def test_c_abi_argument_validation(emu_lib):
    """Null handle, nq < 0, min_count outside [0, K], k outside [1, 32], null buffers with rows to write:
    DSK_ERR_INVALID.  nq == 0 (or an empty index, for neighbors) with null buffers is a valid no-op."""
    lib, k = emu_lib, 32
    buf = _aligned(np.zeros(4096, dtype=np.int64))
    assert lib.dsk_lsh_query_topk(None, _p(buf), 1, 0, 4, _p(buf), _p(buf), None) == DSK_ERR_INVALID
    assert b"null handle" in lib.dsk_last_error()
    assert lib.dsk_lsh_neighbors(None, 0, 4, _p(buf), _p(buf), None) == DSK_ERR_INVALID
    assert b"null handle" in lib.dsk_last_error()
    ix = _EmuTIndex(lib, k, 8, 4, 20)
    try:
        assert lib.dsk_lsh_neighbors(ix.h, 0, 4, None, None, None) == DSK_OK            # empty index
        assert lib.dsk_lsh_neighbors(ix.h, 0, 0, None, None, None) == DSK_ERR_INVALID   # k is checked all the same
        ix.insert(np.arange(3 * k, dtype=np.uint32).reshape(3, k) % 5)
        q = lambda nq, mc, kk, a, b_, c: lib.dsk_lsh_query_topk(ix.h, a, nq, mc, kk, b_, c, None)  # noqa: E731
        nb = lambda mc, kk, b_, c: lib.dsk_lsh_neighbors(ix.h, mc, kk, b_, c, None)           # noqa: E731
        for kk in (0, 33, -1, 1 << 20):
            assert q(1, 0, kk, _p(buf), _p(buf), _p(buf)) == DSK_ERR_INVALID and b"k must be" in lib.dsk_last_error()
            assert nb(0, kk, _p(buf), _p(buf)) == DSK_ERR_INVALID and b"k must be" in lib.dsk_last_error()
        for mc in (-1, k + 1, -(1 << 31)):
            assert q(1, mc, 4, _p(buf), _p(buf), _p(buf)) == DSK_ERR_INVALID and b"min_count" in lib.dsk_last_error()
            assert nb(mc, 4, _p(buf), _p(buf)) == DSK_ERR_INVALID and b"min_count" in lib.dsk_last_error()
        assert q(-1, 0, 4, _p(buf), _p(buf), _p(buf)) == DSK_ERR_INVALID and b"nq must be" in lib.dsk_last_error()
        for args in ((None, _p(buf), _p(buf)), (_p(buf), None, _p(buf)), (_p(buf), _p(buf), None)):
            assert q(1, 0, 4, *args) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
        for args in ((None, _p(buf)), (_p(buf), None)):
            assert nb(0, 4, *args) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
        assert q(0, 0, 4, None, None, None) == DSK_OK
        assert q(1, k, 1, _p(buf), _p(buf), _p(buf)) == DSK_OK and q(1, 0, 32, _p(buf), _p(buf), _p(buf)) == DSK_OK
        assert nb(k, 32, _p(buf), _p(buf)) == DSK_OK
    finally:
        ix.close()


# ---- reference parity (tests/golden/lsh_topk.npz) ------------------------------------------------------------------------
def _golden_cases(g):
    for kk in g["ks"].tolist():
        for j, t in enumerate(g["thresholds"].tolist()):
            yield kk, (None if t < 0 else t), "k%d_t%d" % (kk, j)


def test_oracle_is_the_reference(golden):
    """DictLSH.query + oracle_np.jaccard, sorted by (-eq, d) and cut at k, give the reference's lists and MinHash.jaccard
    values, for held-out queries and for the indexed documents without themselves."""
    g, sig = golden("lsh_topk"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    alive = np.ones(len(sig), dtype=bool)
    ref = _oracle_index(sig, alive, 128, b, r)
    qsig = g["qsig"]
    for kk, t, tag in _golden_cases(g):
        for which, dicts in (("q", _want(ref, sig, qsig, t)), ("s", _nbr_dicts(ref, sig, t, alive))):
            idx, eq = _topk(dicts, kk)
            assert np.array_equal(idx, g["%s_%s_idx" % (which, tag)]), (which, tag)
            assert np.array_equal(np.where(eq >= 0, eq / 128.0, -1.0), g["%s_%s_jac" % (which, tag)]), (which, tag)
    full = g["q_k32_t0_idx"]
    assert (full >= 0).sum(1).max() >= 3 and ((full >= 0).sum(1) == 0).any() and (g["s_k5_t2_idx"][:, 0] >= 0).any()
    assert (g["s_k1_t0_idx"][:, 0] > np.arange(len(sig))).any()              # neighbours above i as well as below


def test_golden_topk(be, golden):
    """The library gives the reference's sorted and cut lists, with MinHash.jaccard * K as eq."""
    g, sig = golden("lsh_topk"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    ix = be.index(128, b, r, len(sig))
    try:
        ix.insert(sig)
        for kk, t, tag in _golden_cases(g):
            for which, (idx, eq) in (("q", ix.query_topk(g["qsig"], kk, t)), ("s", ix.neighbors(kk, t))):
                assert np.array_equal(idx, g["%s_%s_idx" % (which, tag)]), (which, tag)
                assert np.array_equal(np.where(eq >= 0, eq / 128.0, -1.0), g["%s_%s_jac" % (which, tag)]), (which, tag)
    finally:
        ix.close()


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_api_errors_and_outputs():
    """k outside [1, 32] or not an integer raises ValueError; signature errors are query()'s; to_host=False returns CUDA
    int32 tensors of shape [Q, k] / [n, k]."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(5)
    k = 64
    rows = _low_entropy(rs, 300, k, 3)
    ix = dsk.GpuLSH(num_perm=k, params=(16, 4), capacity=300)
    ix.insert(rows)
    q = _perturb(rs, rows[:50], 0.1, 3)
    for bad in (0, 33, -1, 1.0, True, "3", None):
        with pytest.raises(ValueError, match="k must be"):
            ix.query_topk(q, bad)
        with pytest.raises(ValueError, match="k must be"):
            ix.neighbors(bad)
    with pytest.raises(ValueError, match="Expecting minhash with length"):
        ix.query_topk(np.zeros((2, k + 1), dtype=np.uint32), 3)
    with pytest.raises(TypeError):
        ix.query_topk(torch.zeros((2, k), dtype=torch.int64, device="cuda"), 3)
    for fn in (lambda: ix.query_topk(q, 3, 1.5), lambda: ix.neighbors(3, -0.1)):
        with pytest.raises(ValueError):
            fn()
    ti, te = ix.query_topk(torch.from_numpy(q.view(np.int32)).cuda(), np.int64(7), 0.3, to_host=False)
    assert ti.is_cuda and ti.dtype == torch.int32 and te.dtype == torch.int32 and tuple(ti.shape) == (50, 7)
    ni, ne = ix.neighbors(32, to_host=False)
    assert ni.is_cuda and ni.dtype == torch.int32 and tuple(ne.shape) == (300, 32)
    assert np.array_equal(ti.cpu().numpy(), ix.query_topk(q, 7, 0.3)[0])


@pytest.mark.gpu
def test_weighted_python_inputs():
    """On a weighted index query_topk takes [N, ss, 2] numpy rows, CUDA tensors and WeightedMinHash lists alike."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(3)
    ss = 16
    rows = np.stack([rs.randint(0, 3, size=(200, ss)), rs.randint(-1, 1, size=(200, ss))], axis=-1).astype(np.int64)
    ix = dsk.GpuLSH(num_perm=ss, params=(4, 4), capacity=200, weighted=True)
    ix.insert(rows)
    want = ix.query_topk(rows[:20], 9, 0.5)
    for form in (torch.from_numpy(rows[:20]).cuda(), [dsk.WeightedMinHash(1, r) for r in rows[:20]]):
        got = ix.query_topk(form, 9, 0.5)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    ni, ne = ix.neighbors(9, 0.5)
    si, se = ix.query_topk(rows, 10, 0.5)
    for i in range(len(rows)):
        keep = si[i] != i
        assert np.array_equal(si[i][keep][:9], ni[i]) and np.array_equal(se[i][keep][:9], ne[i])


def _segmented_topk(rows, idx, eq, n_rows, n_idx, k, K):
    """(row, idx, eq) triples on the device -> [n_rows, k] idx / eq sorted by (-eq, idx) per row: the torch flow."""
    import torch
    key = (rows.long() * (K + 1) + (K - eq.long())) * n_idx + idx.long()
    key, order = torch.sort(key)
    rows, idx, eq = rows[order].long(), idx[order], eq[order]
    start = torch.searchsorted(rows, torch.arange(n_rows, device=rows.device))
    rank = torch.arange(len(rows), device=rows.device) - start[rows]
    sel = rank < k
    oi = torch.full((n_rows, k), -1, dtype=torch.int32, device=rows.device)
    oe = torch.full((n_rows, k), -1, dtype=torch.int32, device=rows.device)
    oi[rows[sel], rank[sel]] = idx[sel].int()
    oe[rows[sel], rank[sel]] = eq[sel].int()
    return oi, oe


@pytest.mark.gpu
def test_c3_scale_one_million_documents_100k_queries():
    """The C3 workload at 1M documents (128 tokens, K = 256, LSH(0.8)) built through insert_tokens with planted
    near-duplicates, and 100k fresh queries: query_topk(10, 0.5) equals query_jaccard(0.5) + a torch segmented top-k, and
    neighbors(10, 0.5) equals the symmetrised candidate_pairs(0.5) sorted the same way."""
    import torch
    import datasketch_b200 as dsk
    from datasketch_b200.minhash import _make_permutations
    n, t, K, nq, k = 1_000_000, 128, 256, 100_000, 10
    perms = _make_permutations(K, 1)
    g = torch.Generator(device="cuda").manual_seed(7)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, t), dtype=torch.int32, device="cuda", generator=g)
    dup = torch.randint(0, n, (n // 5,), device="cuda", generator=g)            # 20 % near-copies of other documents
    dst = torch.randint(0, n, (n // 5,), device="cuda", generator=g)
    keep = torch.rand((n // 5, t), device="cuda", generator=g) < 0.05
    tok[dst] = torch.where(keep, tok[dst], tok[dup])
    off = torch.arange(0, (n + 1) * t, t, dtype=torch.int64, device="cuda")
    ix = dsk.GpuLSH(threshold=0.8, num_perm=K, capacity=n)
    ix.insert_tokens(tok.view(-1), off, n * t, perms)
    qtok = torch.randint(-2 ** 31, 2 ** 31 - 1, (nq, t), dtype=torch.int32, device="cuda", generator=g)
    src = torch.randint(0, n, (nq // 2,), device="cuda", generator=g)
    mask = torch.rand((nq // 2, t), device="cuda", generator=g) < 0.1
    qtok[:nq // 2] = torch.where(mask, qtok[:nq // 2], tok[src])
    qoff = torch.arange(0, (nq + 1) * t, t, dtype=torch.int64, device="cuda")
    qsig = dsk.engine.bulk_signatures_device(qtok.view(-1), qoff, nq * t, perms)

    ptr, idx, eq = ix.query_jaccard(qsig, 0.5, to_host=False)
    rows = torch.repeat_interleave(torch.arange(nq, device="cuda"), ptr[1:] - ptr[:-1])
    wi, we = _segmented_topk(rows, idx, eq, nq, n, k, K)
    gi, ge = ix.query_topk(qsig, k, 0.5, to_host=False)
    assert int((wi[:, 0] >= 0).sum()) >= nq // 4
    assert torch.equal(gi, wi) and torch.equal(ge, we)

    ptr, idx, eq = ix.candidate_pairs(0.5, to_host=False)
    i = torch.repeat_interleave(torch.arange(n, device="cuda"), ptr[1:] - ptr[:-1])
    wi, we = _segmented_topk(torch.cat([i, idx.long()]), torch.cat([idx, i.int()]), torch.cat([eq, eq]), n, n, k, K)
    gi, ge = ix.neighbors(k, 0.5, to_host=False)
    assert int((wi[:, 0] >= 0).sum()) >= n // 10
    assert torch.equal(gi, wi) and torch.equal(ge, we)
