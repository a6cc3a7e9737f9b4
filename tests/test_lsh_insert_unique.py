"""GpuLSH.insert_unique: insert the rows of a batch that have no near-duplicate yet, as the streaming dedup loop does.

The loop (lsh.py:370-432 query, :326-347 insert, minhash.py:299-324 jaccard) runs over the batch in order::

    for j, m in enumerate(batch):
        if not [d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]:
            lsh.insert(n0 + kept_so_far, m)

``insert_unique(batch, t)`` returns ``(kept, match, eq)``: the loop's decision per row, and for a dropped row the candidate
of the loop's query with the largest eq (the smallest document number among equal ones, numbered as after the call).
The kept rows become documents n0, n0 + 1, ... in batch order.

The oracle is that loop over oracle_np.DictLSH + oracle_np.jaccard, with test_lsh_remove.py's MinHashLSH.remove for the
removed documents; tests/golden/lsh_insert_unique.npz (oracle/gen_golden_lsh_insert_unique.py) pins it to the reference's
own loop.  After every call the index is compared with a fresh one into which the oracle's kept rows were inserted in
order (query, candidate_pairs, duplicate_clusters).  The two backends are those of test_lsh_query_jaccard.py: ``emu``,
the whole library on the emulation shim driven through its C-ABI, and ``gpu``, the Python API on the H100.
"""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle_clib as oc
from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402
from test_lsh_self_join import _aligned, _low_entropy, _min_count, _p  # noqa: E402
from test_lsh_remove import _oracle_index, _state  # noqa: E402
from test_lsh_query_jaccard import _EmuQIndex, _GpuQIndex, _perturb  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
DSK_OK, DSK_ERR_INVALID = 0, 1


# ---- backends ----------------------------------------------------------------------------------------------------------
class _EmuUIndex(_EmuQIndex):
    """The emulated library through its C-ABI: count -> scan -> commit, as GpuLSH.insert_unique runs them."""

    def __init__(self, lib, k, b, r, capacity):
        super().__init__(lib, k, b, r, capacity)
        self.capacity = capacity

    def insert_unique(self, sig, min_jaccard=None):
        """(kept, match, eq), or None when the library refused the call (capacity): the index is then unchanged."""
        lib, sig, mc = self.lib, _aligned(np.asarray(sig, dtype=np.uint32).reshape(-1, self.k)), _min_count(min_jaccard,
                                                                                                           self.k)
        n = len(sig)
        ws_bytes = int(lib.dsk_lsh_unique_workspace_size(self.h, n))
        ws = _aligned(np.zeros(max(ws_bytes, 1), dtype=np.uint8))
        counts, ptr = np.full(n + 1, -7, dtype=np.int64), np.zeros(n + 1, dtype=np.int64)
        scratch = np.zeros(n // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_unique_count(self.h, _p(sig), n, mc, _p(ws), ws_bytes, _p(counts), None) == 0, \
            lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), n, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        pidx, peq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        kept = np.full(max(n, 1), 7, dtype=np.uint8)
        match, eq = np.full(max(n, 1), -7, dtype=np.int32), np.full(max(n, 1), -7, dtype=np.int32)
        ins = ctypes.c_int64(-7)
        rc = lib.dsk_lsh_unique_commit(self.h, _p(sig), n, mc, _p(ws), ws_bytes, _p(ptr), _p(pidx), _p(peq), _p(kept),
                                       _p(match), _p(eq), ctypes.byref(ins), None)
        if rc != 0:
            assert rc == DSK_ERR_INVALID and b"capacity" in lib.dsk_last_error()
            return None
        assert ins.value == int(kept[:n].sum())
        self.n += ins.value
        return kept[:n].astype(bool), match[:n], eq[:n]

    def size(self):
        size = ctypes.c_int64()
        assert self.lib.dsk_lsh_size(self.h, ctypes.byref(size), None) == 0
        return size.value


class _Emu:
    name = "emu"

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuUIndex(self.lib, k, b, r, capacity)


class _GpuUIndex(_GpuQIndex):
    def __init__(self, dsk, k, b, r, capacity):
        super().__init__(dsk, k, b, r, capacity)
        self.k = k

    def insert_unique(self, sig, min_jaccard=None):
        sig = np.ascontiguousarray(np.asarray(sig, dtype=np.uint32).reshape(-1, self.k))
        keys = ["row%d" % j for j in range(len(sig))]
        n0, keys0 = len(self.ix), list(self.ix.keys)
        try:
            kept, match, eq = self.ix.insert_unique(sig, min_jaccard, keys=keys)
        except ValueError as exc:
            assert "capacity" in str(exc)
            assert len(self.ix) == n0 and self.ix.keys == keys0
            return None
        assert kept.dtype == bool and match.dtype == np.int32 and eq.dtype == np.int32
        assert self.ix.keys == keys0 + [kk for kk, kp in zip(keys, kept) if kp]
        self.ix.keys = keys0 + [None] * int(kept.sum())        # the wrapper's index keeps no real keys beyond the check
        assert len(self.ix) == n0 + int(kept.sum())
        return kept, match, eq

    def size(self):
        return len(self.ix)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk

    def index(self, k, b, r, capacity):
        return _GpuUIndex(self.dsk, k, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
def _loop(rows, alive, batch, k, b, r, t):
    """The streaming loop over DictLSH: (kept, match, eq) and the kept rows in batch order."""
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1, k)
    ref = _oracle_index(rows, alive, k, b, r)
    held = list(rows)
    kept, match, eq, new = [], [], [], []
    for m in np.asarray(batch, dtype=np.uint64).reshape(-1, k):
        cand = {d: int(np.count_nonzero(m == held[d])) for d in ref.query(m) if t is None or o.jaccard(m, held[d]) >= t}
        if cand:
            e, d = min((-e, d) for d, e in cand.items())
            kept.append(False)
            match.append(d)
            eq.append(-e)
        else:
            ref.insert(len(held), m)
            held.append(m)
            new.append(m)
            kept.append(True)
            match.append(-1)
            eq.append(-1)
    return (np.array(kept, dtype=bool), np.array(match, dtype=np.int64), np.array(eq, dtype=np.int64),
            np.array(new, dtype=np.uint32).reshape(-1, k))


class _Model:
    """What the index must hold: every row inserted (removed ones included, until compact) and the alive mask."""

    def __init__(self, k):
        self.k = k
        self.rows = np.zeros((0, k), dtype=np.uint32)
        self.alive = np.zeros(0, dtype=bool)

    def add(self, rows):
        rows = np.asarray(rows, dtype=np.uint32).reshape(-1, self.k)
        self.rows = np.concatenate([self.rows, rows])
        self.alive = np.concatenate([self.alive, np.ones(len(rows), dtype=bool)])


def _fresh(be, model, k, b, r):
    """A fresh index of the same backend: the model's rows inserted in order and the removed ones removed."""
    fx = be.index(k, b, r, max(len(model.rows), 1))
    if len(model.rows):
        fx.insert(model.rows)
    gone = np.flatnonzero(~model.alive)
    if len(gone):
        fx.remove(gone)
    return fx


def _unique(be, ix, model, batch, t, k, b, r, probe=None, thresholds=(None, 0.5)):
    """insert_unique(batch, t) against the loop; then the index against a fresh one holding the loop's result."""
    batch = np.asarray(batch, dtype=np.uint32).reshape(-1, k)
    w_kept, w_match, w_eq, new = _loop(model.rows, model.alive, batch, k, b, r, t)
    got = ix.insert_unique(batch, t)
    assert got is not None
    kept, match, eq = got
    assert np.array_equal(kept, w_kept), t
    assert np.array_equal(match.astype(np.int64), w_match), t
    assert np.array_equal(eq.astype(np.int64), w_eq), t
    model.add(new)
    assert ix.size() == len(model.rows)
    probe = np.concatenate([model.rows, batch]) if probe is None else probe
    fx = _fresh(be, model, k, b, r)
    try:
        assert _state(ix, probe, thresholds) == _state(fx, probe, thresholds)
    finally:
        fx.close()
    return kept, match, eq


def _drift_chain(rs, n, k, b, r):
    """n rows where row i and row i + 1 share half of the bands (the even ones for even i, the odd ones for odd i) and
    rows two apart share no band: eq = (b / 2) * r between neighbours, far less between any other two."""
    rows = rs.randint(0, 1 << 32, size=(n, k), dtype=np.uint64).astype(np.uint32)
    for j in range(b):
        vals = rs.randint(0, 1 << 32, size=(n // 2 + 2, r), dtype=np.uint64).astype(np.uint32)
        grp = (np.arange(n) + (j % 2)) // 2
        rows[:, j * r:(j + 1) * r] = vals[grp]
    return rows


# ---- cases -------------------------------------------------------------------------------------------------------------
def test_drift_chain_differs_from_duplicate_clusters(be):
    """a ~ b ~ c ~ ... with rows two apart unrelated: the loop keeps every other row, the components keep only the first."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(1)
    chain = _drift_chain(rs, 9, k, b, r)
    for t in (None, 0.5):
        ix, model = be.index(k, b, r, 20), _Model(k)
        try:
            kept, match, eq = _unique(be, ix, model, chain, t, k, b, r)
            assert kept.tolist() == [j % 2 == 0 for j in range(9)]
            assert match.tolist() == [-1 if j % 2 == 0 else j // 2 for j in range(9)]   # numbers of the kept rows 0, 2, ...
            assert np.all(eq[1::2] == (b // 2) * r)
            fx = be.index(k, b, r, 20)                                  # the whole chain in one index: one component
            fx.insert(chain)
            labels = np.asarray(fx.clusters(t))
            fx.close()
            assert labels.tolist() == [0] * 9
            roots = labels == np.arange(9)
            assert roots.sum() == 1 and kept.sum() == 5 and not np.array_equal(roots, kept)
        finally:
            ix.close()


def test_long_drift_chain_many_rounds(be):
    """A chain of 2,100 rows behind an index that already holds its head: every decision waits for the one before it,
    so the resolution takes about as many rounds as the chain is long, over more rows than one resolving sweep."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(2)
    n = 2100
    chain = _drift_chain(rs, n + 1, k, b, r)
    other = rs.randint(0, 1 << 32, size=(50, k), dtype=np.uint64).astype(np.uint32)
    ix, model = be.index(k, b, r, 200 + n), _Model(k)
    try:
        ix.insert(np.concatenate([other, chain[:1]]))
        model.add(np.concatenate([other, chain[:1]]))
        batch = np.concatenate([chain[1:], other[:5]])
        kept, match, _ = _unique(be, ix, model, batch, 0.5, k, b, r, probe=batch[::7])
        assert kept[:n].tolist() == [j % 2 == 1 for j in range(n)] and not kept[n:].any()
        assert match[0] == len(other) and match[2] == len(other) + 1
    finally:
        ix.close()


def test_within_batch_bucket_of_exact_copies(be):
    """Hundreds of exact copies in one batch (one bucket per band with all of them): the first is kept, every other copy
    is dropped with the first as its match (eq = K); a copy of an indexed row is dropped by the index instead."""
    k, b, r = 64, 16, 4
    rs = np.random.RandomState(3)
    rows = rs.randint(0, 1 << 32, size=(4, k), dtype=np.uint64).astype(np.uint32)
    copies = 200 if be.name == "emu" else 700
    batch = np.concatenate([rows[3:4], np.repeat(rows[:1], copies, 0), np.repeat(rows[1:2], 20, 0),
                            np.repeat(rows[2:3], 5, 0)])
    batch = batch[rs.permutation(len(batch))]
    ix, model = be.index(k, b, r, 10), _Model(k)
    try:
        ix.insert(rows[2:3])
        model.add(rows[2:3])
        for t in (None,) if be.name == "emu" else (None, 1.0):
            kept, match, eq = _unique(be, ix, model, batch, t, k, b, r, probe=rows, thresholds=(None,))
            assert kept.sum() == (3 if t is None else 0)
            assert np.all(eq[~kept] == k)
    finally:
        ix.close()


@pytest.mark.parametrize("k,b,r,vals", [(32, 8, 4, 3), (100, 33, 3, 4)])
def test_low_entropy_exact_thresholds(be, k, b, r, vals):
    """Big buckets and (b = 33) a second lane round; the batch mixes indexed rows, perturbed ones and fresh ones, at no
    threshold, 0.0, 1.0 and the exact boundaries c / K and (c + 1) / K."""
    rs = np.random.RandomState(k + b)
    n = 60 if be.name == "emu" else 1500
    nb = 60 if be.name == "emu" else 1500
    sig = _low_entropy(rs, n, k, vals)
    third = nb // 3
    batch = np.concatenate([sig[rs.choice(n, third)], _perturb(rs, sig[rs.choice(n, third)], 0.15, vals),
                            _low_entropy(rs, nb - 2 * third, k, vals)])
    batch = batch[rs.permutation(len(batch))]
    c = k // 3
    for t in (None, 0.0, 1.0, c / k, (c + 1) / k):
        ix, model = be.index(k, b, r, n + nb), _Model(k)
        try:
            ix.insert(sig[:n // 2])
            model.add(sig[:n // 2])
            kept, _, _ = _unique(be, ix, model, batch, t, k, b, r, thresholds=(None, c / k))
            if t == 1.0:
                assert 0 < kept.sum() < len(batch)
        finally:
            ix.close()


def test_index_drops_rows_that_also_match_kept_batch_rows(be):
    """A row dropped by the index that also matches earlier kept rows of the batch: the match is the best of both, and
    on an eq tie the indexed document (the smaller number) wins; a batch row with a larger eq wins over the index."""
    k, b, r = 64, 16, 4
    rs = np.random.RandomState(5)
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)

    def variant(bands_broken, extra):
        d = q.copy()
        pos = [j * r for j in bands_broken] + list(extra)
        d[pos] += 1 + rs.randint(0, 1000, size=len(pos)).astype(np.uint32)
        return d
    noise = rs.randint(0, 1 << 32, size=(3, k), dtype=np.uint64).astype(np.uint32)
    x = variant(range(0, 8), [])                            # indexed, eq(q, x) = K - 8, shares bands 8..15 with q
    a = variant(range(8, 16), [])                           # batch, eq(q, a) = K - 8 (tie with x), shares 0..7
    a2 = variant(range(8, 15), [])                          # batch, eq(q, a2) = K - 7, shares band 15 with x
    y = variant(range(0, 8), [15 * r + 1])                  # indexed, eq(q, y) = K - 9
    ix, model = be.index(k, b, r, 20), _Model(k)
    try:
        ix.insert(np.concatenate([noise, x[None]]))
        model.add(np.concatenate([noise, x[None]]))
        kept, match, eq = _unique(be, ix, model, np.stack([a, q]), (k - 8) / k, k, b, r)
        assert kept.tolist() == [True, False] and match.tolist() == [-1, 3] and eq.tolist() == [-1, k - 8]
        kept, match, eq = _unique(be, ix, model, np.stack([a2, q]), (k - 8) / k, k, b, r)
        assert kept.tolist() == [False, False] and match.tolist() == [4, 3]     # a2 ~ a (eq K - 1); q: x ties a
    finally:
        ix.close()
    ix, model = be.index(k, b, r, 20), _Model(k)
    try:
        ix.insert(np.concatenate([noise, y[None]]))
        model.add(np.concatenate([noise, y[None]]))
        kept, match, eq = _unique(be, ix, model, np.stack([a, q]), None, k, b, r)
        assert kept.tolist() == [True, False] and match.tolist() == [-1, 4] and eq.tolist() == [-1, k - 8]
    finally:
        ix.close()


@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_and_the_empty_key(be, head_collides):
    """Tuples that share a band's fingerprint without being equal (hash_model second preimages, bands 0, 31 and 35) and
    the tuple whose fingerprint is the tables' empty key.  The index holds tuple t; the batch holds rows with t and rows
    with its colliding twin t2, in both orders, so each chain of the index and of the batch table mixes the two: a row
    with t2 is no candidate of a row with t, neither against the index nor within the batch."""
    k, b, r = 120, 40, 3
    rs = np.random.RandomState(41 + head_collides)
    base = rs.randint(0, 1 << 32, size=(30, k), dtype=np.uint64).astype(np.uint32)
    batch, want = [], []
    for band in (0, 31, 35):
        sl = slice(band * r, (band + 1) * r)
        for d in rs.permutation(len(base)):
            t2 = hm.second_preimage(base[d, sl], band, rs)
            if t2 is None:
                continue
            x = rs.randint(0, 1 << 32, size=(4, k), dtype=np.uint64).astype(np.uint32)
            first, second = (t2, base[d, sl]) if head_collides else (base[d, sl], t2)
            x[0::2, sl], x[1::2, sl] = first, second
            batch.append(x)
            want += [True, False, False, False] if head_collides else [False, True, False, False]
            break
        else:
            pytest.fail("no second preimage found for band %d" % band)
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, r, rs)
        if e is not None:
            em = rs.randint(0, 1 << 32, size=(3, k), dtype=np.uint64).astype(np.uint32)
            em[:, band * r:(band + 1) * r] = e
            batch.append(em)
            want += [True, False, False]
            break
    else:
        pytest.fail("no empty-key tuple found")
    batch = np.concatenate(batch)
    fp = hm.band_fp(batch, b, r)
    assert len(np.unique(fp)) < fp.size
    ix, model = be.index(k, b, r, len(base) + len(batch)), _Model(k)
    try:
        for row in base:
            ix.insert(row[None])
        model.add(base)
        kept, _, _ = _unique(be, ix, model, batch, None, k, b, r)
        assert kept.tolist() == want
    finally:
        ix.close()


def test_removed_documents_never_drop_a_row(be):
    """Removed chain heads, middles and tails: a batch row whose only near-duplicates were removed is kept, before and
    after compact(); a removed document is never a match."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(7)
    groups, size = 4, 5
    rows = rs.randint(0, 1 << 32, size=(groups * size + 10, k), dtype=np.uint64).astype(np.uint32)
    for g in range(groups):                                      # member j of group g is row j * groups + g
        rows[g:groups * size:groups, 0:r] = rs.randint(0, 1 << 32, size=r, dtype=np.uint64).astype(np.uint32)
    batch = np.concatenate([rows, _perturb(rs, rows, 0.2, 1 << 30)])
    batch[len(rows):, 0:r] = rows[:, 0:r]
    for compact in (False, True):
        ix, model = be.index(k, b, r, 3 * len(rows) + 10), _Model(k)
        try:
            for row in rows:
                ix.insert(row[None])
            model.add(rows)
            gone = [(size - 1) * groups + 0, 2 * groups + 1, 0 * groups + 2] + list(range(3, groups * size, groups))
            ix.remove(gone)
            model.alive[gone] = False
            if compact:
                ix.compact()
                model.rows, model.alive = model.rows[model.alive], model.alive[model.alive]
            kept, match, _ = _unique(be, ix, model, batch, 0.5, k, b, r)
            assert kept[:len(rows)].tolist() == (~model.alive[:len(rows)]).tolist() if not compact else True
            assert np.all(model.alive[match[(match >= 0) & (match < len(model.alive))]])
            assert kept.any() and not kept.all()
        finally:
            ix.close()


def test_rows_from_the_fused_token_insert(be):
    """An index built from tokens (the signature kernel's fused insert epilogue), a batch of near-duplicate documents
    of it with 10 % of the tokens resampled, some fresh ones and copies within the batch."""
    k, b, r = 128, 32, 4
    rs = np.random.RandomState(9)
    n = 80 if be.name == "emu" else 2000
    lens = rs.randint(1, 200, size=n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    perms = o.init_permutations(k, 5)
    sig = oc.minhash_bulk_u32tok(tok, off, perms)
    qtok = tok.copy()
    qtok[rs.rand(len(qtok)) < 0.1] = rs.randint(0, 1 << 32, dtype=np.uint64)
    qsig = oc.minhash_bulk_u32tok(qtok, off, perms)
    fresh = rs.randint(0, 1 << 32, size=(10, k), dtype=np.uint64).astype(np.uint32)
    batch = np.concatenate([qsig, fresh, qsig[:10], fresh[:3]])
    ix, model = be.index(k, b, r, n + len(batch)), _Model(k)
    try:
        ix.insert_tokens(tok, off, perms)
        model.add(sig)
        kept, _, _ = _unique(be, ix, model, batch, 0.7, k, b, r, thresholds=(None, 0.7))
        assert (~kept[:n]).sum() >= n // 4 and kept[n:n + 10].all() and not kept[n + 10:].any()
    finally:
        ix.close()


def test_sizes_empty_all_duplicates_twice_and_capacity(be):
    """An empty index, an empty batch, a batch that is all duplicates (nothing kept), the same batch twice (the second
    call keeps nothing), a capacity that fits exactly, and one exceeded: refused with the index unchanged."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(11)
    rows = rs.randint(0, 1 << 32, size=(6, k), dtype=np.uint64).astype(np.uint32)
    batch = np.concatenate([rows, rows[:3]])                     # 6 distinct + 3 copies: 6 kept into an empty index
    ix, model = be.index(k, b, r, 6), _Model(k)
    try:
        kept, _, _ = _unique(be, ix, model, np.zeros((0, k), dtype=np.uint32), None, k, b, r, probe=rows)
        assert len(kept) == 0 and ix.size() == 0
        kept, match, _ = _unique(be, ix, model, batch, None, k, b, r)    # capacity 6: fits exactly
        assert kept.sum() == 6 and ix.size() == 6 and match[6:].tolist() == [0, 1, 2]
        kept, match, eq = _unique(be, ix, model, batch, None, k, b, r)   # the same batch again: all duplicates
        assert not kept.any() and match.tolist() == [0, 1, 2, 3, 4, 5, 0, 1, 2] and np.all(eq == k)
        before = _state(ix, batch, (None,))
        assert ix.insert_unique(rs.randint(0, 1 << 32, size=(1, k), dtype=np.uint64).astype(np.uint32)) is None
        assert ix.size() == 6 and _state(ix, batch, (None,)) == before
    finally:
        ix.close()
    ix, model = be.index(k, b, r, 8), _Model(k)
    try:
        ix.insert(rows[:5])
        model.add(rows[:5])
        fresh = rs.randint(0, 1 << 32, size=(4, k), dtype=np.uint64).astype(np.uint32)
        assert ix.insert_unique(np.concatenate([rows, fresh]), None) is None   # 5 + 5 kept > 8: refused
        assert ix.size() == 5 and _state(ix, rows, (None,)) == _state(_fresh(be, model, k, b, r), rows, (None,))
        kept, _, _ = _unique(be, ix, model, np.concatenate([rows, fresh[:2], rows]), None, k, b, r)  # 5 + 3 = 8 fits
        assert kept.sum() == 3 and ix.size() == 8
    finally:
        ix.close()


@pytest.mark.parametrize("k", [2048, 4096])
def test_large_k(be, k):
    """K = 2048 and 4096: fewer warps per CTA in both walks."""
    b, r = 16, 4
    rs = np.random.RandomState(k)
    n = 30
    sig = rs.randint(0, 4, size=(n, k)).astype(np.uint32)
    sig[:, b * r:] = rs.randint(0, 1 << 32, size=(n, k - b * r), dtype=np.uint64).astype(np.uint32)
    batch = np.concatenate([sig[:6], _perturb(rs, sig[6:20], 0.3, 4), sig[20:], sig[25:]])
    ix, model = be.index(k, b, r, 2 * n + len(batch)), _Model(k)
    try:
        ix.insert(sig[:10])
        model.add(sig[:10])
        for t in (None, 0.5):
            _unique(be, ix, model, batch, t, k, b, r, probe=batch[::3], thresholds=(None,))
    finally:
        ix.close()


def test_c_abi_argument_validation(emu_lib):
    """Bad handle, n < 0, min_count outside [0, K], a short or misaligned workspace, null buffers with n > 0, and a commit
    that does not follow a count of the same rows and workspace: DSK_ERR_INVALID.  n == 0 with null buffers is a no-op."""
    lib, k = emu_lib, 32
    ix = _EmuUIndex(lib, k, 8, 4, 20)
    sig = _aligned(np.arange(3 * k, dtype=np.uint32).reshape(3, k) % 5)
    n = 3
    try:
        ws_bytes = int(lib.dsk_lsh_unique_workspace_size(ix.h, n))
        assert ws_bytes > 0 and lib.dsk_lsh_unique_workspace_size(None, n) == 0
        assert lib.dsk_lsh_unique_workspace_size(ix.h, -1) == 0 and lib.dsk_lsh_unique_workspace_size(ix.h, 0) == 0
        ws = _aligned(np.zeros(ws_bytes + 64, dtype=np.uint8))
        buf = _aligned(np.zeros(256, dtype=np.int64))
        ins = ctypes.c_int64()

        def count(h=ix.h, s=_p(sig), nn=n, mc=0, w=_p(ws), wb=ws_bytes, c=_p(buf)):
            return lib.dsk_lsh_unique_count(h, s, nn, mc, w, wb, c, None)

        def commit(h=ix.h, s=_p(sig), nn=n, mc=0, w=_p(ws), wb=ws_bytes, bufs=None, hi=ctypes.byref(ins)):
            bufs = [_p(buf)] * 6 if bufs is None else bufs
            return lib.dsk_lsh_unique_commit(h, s, nn, mc, w, wb, *bufs, hi, None)

        for fn in (count, commit):
            assert fn(h=None) == DSK_ERR_INVALID and b"null handle" in lib.dsk_last_error()
            assert fn(nn=-1) == DSK_ERR_INVALID and b"n must be" in lib.dsk_last_error()
            for mc in (-1, k + 1):
                assert fn(mc=mc) == DSK_ERR_INVALID and b"min_count" in lib.dsk_last_error()
            assert fn(wb=ws_bytes - 1) == DSK_ERR_INVALID and b"workspace" in lib.dsk_last_error()
            misaligned = ctypes.c_void_p(ws.ctypes.data + 8)
            assert fn(w=misaligned) == DSK_ERR_INVALID and b"workspace" in lib.dsk_last_error()
            assert fn(s=None) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
            assert fn(w=None) == DSK_ERR_INVALID
        assert count(c=None) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
        for j in range(6):
            bufs = [_p(buf)] * 6
            bufs[j] = None
            assert commit(bufs=bufs) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
        assert commit(hi=None) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error()
        assert commit() == DSK_ERR_INVALID and b"dsk_lsh_unique_count" in lib.dsk_last_error()   # no count before
        assert count() == DSK_OK
        other = _aligned(sig.copy())
        assert commit(s=_p(other)) == DSK_ERR_INVALID and b"dsk_lsh_unique_count" in lib.dsk_last_error()
        assert count() == DSK_OK
        ws2 = _aligned(np.zeros(ws_bytes, dtype=np.uint8))
        assert commit(w=_p(ws2)) == DSK_ERR_INVALID and b"dsk_lsh_unique_count" in lib.dsk_last_error()
        assert count() == DSK_OK
        assert commit(mc=1) == DSK_ERR_INVALID and b"dsk_lsh_unique_count" in lib.dsk_last_error()
        assert count() == DSK_OK
        ix.insert(sig[:1])                                                  # the index changed in between
        assert commit() == DSK_ERR_INVALID and b"dsk_lsh_unique_count" in lib.dsk_last_error()
        assert ix.size() == 1
        assert lib.dsk_lsh_unique_count(ix.h, None, 0, 0, None, 0, None, None) == DSK_OK
        assert lib.dsk_lsh_unique_commit(ix.h, None, 0, 0, None, 0, *[None] * 6, None, None) == DSK_OK
        assert ix.size() == 1
    finally:
        ix.close()


def test_thread_sanitizer_resolution():
    """The greedy resolution under ThreadSanitizer (tests/emu/emu_tsan_unique_main.cpp, linked with the whole emulated
    library): statuses written and read by concurrent lanes through relaxed atomics, a drift chain resolved over many
    rounds in the single resolving CTA, checked against a serial loop."""
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = os.path.join(EMU, "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "emu_tsan_unique")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-ffp-contract=off", "-fsanitize=thread", "-DDSK_EMU",
                            "-I" + EMU, "-o", exe, os.path.join(EMU, "emu_capi.cpp"),
                            os.path.join(EMU, "emu_tsan_unique_main.cpp")], capture_output=True, text=True)
    if build.returncode != 0:
        pytest.skip("ThreadSanitizer build unavailable: " + build.stderr[-300:])
    env = dict(os.environ, TSAN_OPTIONS="history_size=7 halt_on_error=1 exitcode=66")
    run = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=1800)
    assert "ThreadSanitizer" not in run.stderr, run.stderr[-3000:]
    assert run.returncode == 0, run.stdout + run.stderr[-2000:]
    assert run.stdout.count("identical") == 3, run.stdout


# ---- reference parity (tests/golden/lsh_insert_unique.npz) ----------------------------------------------------------------
def test_oracle_is_the_reference(golden):
    """The loop over DictLSH + oracle_np.jaccard gives the reference's own loop (MinHashLSH.query, MinHash.jaccard,
    MinHashLSH.insert) over a held-out batch against lsh.npz's 300 documents."""
    g, sig = golden("lsh_insert_unique"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    batch = g["batch"]
    alive = np.ones(len(sig), dtype=bool)
    for j, t in enumerate(g["thresholds"].tolist()):
        t = None if t < 0 else t
        kept, match, eq, _ = _loop(sig, alive, batch, 128, b, r, t)
        assert kept.tolist() == g["kept%d" % j].astype(bool).tolist(), t
        assert match.tolist() == g["match%d" % j].tolist(), t
        assert (eq / 128.0).tolist() == [x if x >= 0 else -1 / 128.0 for x in g["jaccard%d" % j].tolist()], t
        assert 0 < kept.sum() < len(batch)


def test_golden_insert_unique(be, golden):
    """The library keeps the rows the reference's loop keeps, with its matches and MinHash.jaccard * K as eq."""
    g, sig = golden("lsh_insert_unique"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    batch = g["batch"]
    for j, t in enumerate(g["thresholds"].tolist()):
        t = None if t < 0 else t
        ix = be.index(128, b, r, len(sig) + len(batch))
        try:
            ix.insert(sig)
            kept, match, eq = ix.insert_unique(batch, t)
            assert kept.tolist() == g["kept%d" % j].astype(bool).tolist(), t
            assert match.tolist() == g["match%d" % j].tolist(), t
            assert [e / 128.0 if e >= 0 else -1.0 for e in eq.tolist()] == g["jaccard%d" % j].tolist(), t
        finally:
            ix.close()


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_api_errors_and_outputs():
    """Wrong K, non-32-bit tensors, a bad min_jaccard and a keys list of the wrong length raise before anything changes;
    to_host=False returns CUDA tensors; keys are appended for the kept rows only."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(4)
    k = 64
    rows = rs.randint(0, 1 << 32, size=(20, k), dtype=np.uint64).astype(np.uint32)
    ix = dsk.GpuLSH(num_perm=k, params=(16, 4), capacity=100)
    ix.insert(rows[:5], keys=list("abcde"))
    with pytest.raises(ValueError, match="Expecting minhash with length"):
        ix.insert_unique(np.zeros((2, k + 1), dtype=np.uint32))
    with pytest.raises(TypeError):
        ix.insert_unique(torch.zeros((2, k), dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        ix.insert_unique(rows, 1.5)
    with pytest.raises(ValueError, match="one key per row"):
        ix.insert_unique(rows, keys=["x"])
    assert len(ix) == 5 and ix.keys == list("abcde")
    kept, match, eq = ix.insert_unique(torch.from_numpy(rows.view(np.int32)).cuda(), 0.5, keys=range(20), to_host=False)
    assert kept.is_cuda and kept.dtype == torch.bool and match.dtype == torch.int32 and eq.dtype == torch.int32
    assert kept.cpu().tolist() == [False] * 5 + [True] * 15 and match.cpu().tolist()[:5] == [0, 1, 2, 3, 4]
    assert len(ix) == 20 and ix.keys == list("abcde") + list(range(5, 20))
    kept, _, _ = ix.insert_unique(rows)
    assert not kept.any() and len(ix) == 20


@pytest.mark.gpu
def test_c3_scale_one_million_documents_100k_batch():
    """The C3 workload at 1M documents (128 tokens, K = 256, LSH(0.8)) built through insert_tokens, and a batch of 100k
    fresh documents: perturbed copies of indexed ones, copies and drift chains within the batch, unrelated ones.
    insert_unique(0.8) equals the two-step flow: query_best against the index, a temporary GpuLSH over the batch, its
    candidate_pairs(0.8), the greedy loop over the pairs on the host, then insert of the survivors."""
    import torch
    import datasketch_b200 as dsk
    from datasketch_b200.minhash import _make_permutations
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_configs import c3_unique_batch, two_step_unique
    n, t, k, nb = 1_000_000, 128, 256, 100_000
    perms = _make_permutations(k, 1)
    g = torch.Generator(device="cuda").manual_seed(5)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, t), dtype=torch.int32, device="cuda", generator=g)
    off = torch.arange(0, (n + 1) * t, t, dtype=torch.int64, device="cuda")
    cap = n + nb
    a = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=cap)
    a.insert_tokens(tok.view(-1), off, n * t, perms)
    btok = c3_unique_batch(tok, nb, g)
    boff = torch.arange(0, (nb + 1) * t, t, dtype=torch.int64, device="cuda")
    bsig = dsk.engine.bulk_signatures_device(btok.view(-1), boff, nb * t, perms)
    kept, match, eq = a.insert_unique(bsig, 0.8)
    b = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=cap)
    b.insert_tokens(tok.view(-1), off, n * t, perms)
    w_kept, w_match, w_eq = two_step_unique(b, bsig, 0.8)
    assert 0.2 * nb < kept.sum() < 0.9 * nb
    assert np.array_equal(kept, w_kept) and np.array_equal(match, w_match) and np.array_equal(eq, w_eq)
    assert len(a) == len(b) == n + int(kept.sum())
    probe = bsig[::50]
    pa, ia = a.query(probe)
    pb, ib = b.query(probe)
    assert np.array_equal(pa, pb) and [set(ia[pa[q]:pa[q + 1]]) for q in range(len(pa) - 1)] == \
        [set(ib[pb[q]:pb[q + 1]]) for q in range(len(pb) - 1)]
