"""GpuLSH.remove / alive / compact: removing documents from a device-resident LSH index, and compacting it.

After a removal ``query`` never returns the document, ``candidate_pairs`` pairs nothing with it and ``duplicate_clusters``
labels it -1 (MinHashLSH.remove, lsh.py:497-528).  A pair depends only on its two rows, so the pairs and clusters after a
removal are those before it restricted to the remaining documents.  ``compact`` renumbers the remaining documents in their
old order; the index then equals a fresh one into which the remaining rows were inserted in order.

The oracle is the dict-bucket index oracle_np.DictLSH with the removal below (``_DictLSH.remove``, pinned to the
reference's MinHashLSH.remove by tests/golden/lsh_remove.npz, which oracle/gen_golden_lsh_remove.py writes),
oracle_np.jaccard and scipy's connected components over the remaining documents.  The two
backends are those of test_lsh_self_join.py: ``emu``, the whole library on the emulation shim driven through its C-ABI,
and ``gpu``, the Python API on the H100.
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
from test_lsh_self_join import (_EmuIndex, _GpuIndex, _aligned, _components, _low_entropy, _p,  # noqa: E402
                                _pairs_dict)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
DSK_OK, DSK_ERR_INVALID = 0, 1


# ---- backends ----------------------------------------------------------------------------------------------------------
class _EmuRmIndex(_EmuIndex):
    """The emulated library through its C-ABI, with the removal entries."""

    def remove(self, docs):
        """dsk_lsh_remove; returns d_status (out of range, already removed)."""
        d = _aligned(np.asarray(docs, dtype=np.int32).reshape(-1))
        status = np.zeros(2, dtype=np.int64)
        assert self.lib.dsk_lsh_remove(self.h, _p(d), len(d), _p(status), None) == 0, self.lib.dsk_last_error()
        return status

    def alive(self, docs=None):
        d = _aligned(np.arange(self.n, dtype=np.int32) if docs is None else np.asarray(docs, dtype=np.int32).reshape(-1))
        out = np.full(max(len(d), 1), 7, dtype=np.uint8)
        assert self.lib.dsk_lsh_alive(self.h, _p(d), len(d), _p(out), None) == 0, self.lib.dsk_last_error()
        return out[:len(d)].astype(bool)

    def compact(self):
        lib, n = self.lib, self.n
        ws = _aligned(np.zeros(max(int(lib.dsk_lsh_compact_workspace_size(self.h)), 1), dtype=np.uint8))
        remap = np.full(max(n, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_compact(self.h, _p(remap), _p(ws), ws.nbytes, None) == 0, lib.dsk_last_error()
        size = ctypes.c_int64()
        assert lib.dsk_lsh_size(self.h, ctypes.byref(size), None) == 0
        self.n = size.value
        return remap[:n]

    def query(self, sig):
        lib, sig = self.lib, _aligned(np.asarray(sig, dtype=np.uint32))
        nq = len(sig)
        counts, ptr = np.zeros(nq + 1, dtype=np.int64), np.zeros(nq + 1, dtype=np.int64)
        scratch = np.zeros(nq // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_query_count(self.h, _p(sig), nq, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), nq, _p(ptr), _p(scratch), None) == 0
        idx = np.full(max(int(ptr[-1]), 1), -1, dtype=np.int32)
        assert lib.dsk_lsh_query_fill(self.h, _p(sig), nq, _p(ptr), _p(idx), None) == 0, lib.dsk_last_error()
        return ptr, idx[:int(ptr[-1])]

    def try_insert(self, sig):
        """True if the insert was accepted (False: refused, e.g. over capacity)."""
        sig = _aligned(np.asarray(sig, dtype=np.uint32))
        if self.lib.dsk_lsh_insert(self.h, _p(sig), len(sig), None) != 0:
            return False
        self.n += len(sig)
        return True


class _Emu:
    name = "emu"

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuRmIndex(self.lib, k, b, r, capacity)


class _GpuRmIndex(_GpuIndex):
    def remove(self, docs):
        self.ix.remove(docs)

    def alive(self, docs=None):
        return self.ix.alive(docs)

    def compact(self):
        return self.ix.compact()

    def query(self, sig):
        return self.ix.query(np.ascontiguousarray(sig, dtype=np.uint32))

    def try_insert(self, sig):
        try:
            self.ix.insert(np.ascontiguousarray(sig, dtype=np.uint32))
        except ValueError as exc:
            assert "capacity" in str(exc)
            return False
        return True


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk

    def index(self, k, b, r, capacity):
        return _GpuRmIndex(self.dsk, k, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
class _DictLSH(o.DictLSH):
    """oracle_np.DictLSH with MinHashLSH.remove."""

    def remove(self, key):
        """datasketch/lsh.py:509-528: drop the key from each of its buckets, an emptied bucket itself, then the key."""
        if key not in self.keys:
            raise ValueError("The given key does not exist")
        for h, table in zip(self.keys[key], self.hashtables):
            table[h].discard(key)
            if not table.get(h):
                del table[h]
        del self.keys[key]


def _oracle_index(rows, alive, k, b, r):
    """_DictLSH over every row, then _DictLSH.remove of the removed ones (as MinHashLSH.remove would)."""
    ref = _DictLSH(k, b, r)
    rows = np.asarray(rows, dtype=np.uint64)
    for i, row in enumerate(rows):
        ref.insert(i, row)
    for i in np.flatnonzero(~alive).tolist():
        ref.remove(i)
    return ref


def _want_pairs(ref, rows, alive, min_jaccard):
    rows = np.asarray(rows, dtype=np.uint64)
    out = {}
    for i in np.flatnonzero(alive).tolist():
        for d in ref.query(rows[i]):
            if d < i and (min_jaccard is None or o.jaccard(rows[i], rows[d]) >= min_jaccard):
                out[(i, d)] = int(np.count_nonzero(rows[i] == rows[d]))
    return out


def _want_labels(n, alive, pairs):
    labels = _components(n, pairs).astype(np.int64) if n else np.zeros(0, dtype=np.int64)
    labels[~alive] = -1
    return labels


def _csr_sets(ptr, idx):
    return [set(idx[ptr[q]:ptr[q + 1]].tolist()) for q in range(len(ptr) - 1)]


def _state(ix, rows, thresholds):
    """What the index answers: query of every row, and pairs + labels per threshold."""
    got = {"query": _csr_sets(*ix.query(rows)) if len(rows) else []}
    for t in thresholds:
        got[t] = (_pairs_dict(*ix.pairs(t)), np.asarray(ix.clusters(t), dtype=np.int64).tolist())
    return got


def _check(ix, rows, alive, k, b, r, thresholds=(None, 0.5)):
    """Compares query / candidate_pairs / duplicate_clusters with the oracle; returns the state for the compaction check."""
    rows = np.asarray(rows, dtype=np.uint32)
    n = len(rows)
    assert np.array_equal(ix.alive(), alive)
    ref = _oracle_index(rows, alive, k, b, r)
    got = _state(ix, rows, thresholds)
    assert got["query"] == [ref.query(row) for row in rows.astype(np.uint64)]
    for t in thresholds:
        want = _want_pairs(ref, rows, alive, t)
        assert got[t][0] == want, t
        assert np.array_equal(got[t][1], _want_labels(n, alive, want)), t
    return got


def _check_compact(be, ix, rows, alive, k, b, r, before, thresholds=(None, 0.5)):
    """compact(): remap keeps the order; pairs and labels map through it; equal to a fresh index of the remaining rows."""
    rows = np.asarray(rows, dtype=np.uint32)
    remap = np.asarray(ix.compact(), dtype=np.int64)
    want_remap = np.where(alive, np.cumsum(alive) - 1, -1)
    assert np.array_equal(remap, want_remap)
    kept = rows[alive]
    after = _state(ix, kept, thresholds)
    assert np.all(ix.alive())
    assert after["query"] == [{int(remap[d]) for d in before["query"][i]} for i in np.flatnonzero(alive)]
    for t in thresholds:
        pairs, labels = before[t][0], np.asarray(before[t][1], dtype=np.int64)
        assert after[t][0] == {(int(remap[i]), int(remap[d])): e for (i, d), e in pairs.items()}, t
        assert np.array_equal(after[t][1], remap[labels[alive]]), t
    fresh = be.index(k, b, r, max(len(kept), 1))
    try:
        if len(kept):
            fresh.insert(kept)
        assert _state(fresh, kept, thresholds) == after
    finally:
        fresh.close()
    return remap


# ---- cases -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frac", [0.1, 0.5, 1.0])
@pytest.mark.parametrize("k,b,r,vals", [(32, 8, 4, 3), (100, 33, 3, 4)])
def test_low_entropy_remove_random_subset(be, k, b, r, vals, frac):
    """Big buckets, exact duplicates, b > 32 bands (two lane rounds): remove 10 %, 50 % or all of the documents, check,
    compact, check again and against a fresh index of the remaining rows."""
    rs = np.random.RandomState(int(frac * 100) + b)
    n = (150 if b <= 32 else 90) if be.name == "emu" else 2500
    sig = _low_entropy(rs, n, k, vals)
    ix = be.index(k, b, r, n)
    ix.insert(sig[:n // 2])
    ix.insert(sig[n // 2:])
    try:
        alive = np.ones(n, dtype=bool)
        gone = rs.choice(n, int(round(frac * n)), replace=False)
        ix.remove(gone[:len(gone) // 2])
        ix.remove(gone[len(gone) // 2:])
        alive[gone] = False
        before = _check(ix, sig, alive, k, b, r)
        _check_compact(be, ix, sig, alive, k, b, r, before)
    finally:
        ix.close()


def test_removed_at_chain_head_middle_and_tail(be):
    """Members of four buckets inserted one at a time, so each chain runs from the last inserted to the first: remove a
    chain's head, a middle member, its tail, and every member of the fourth bucket."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(3)
    groups, size = 4, 5
    rows = rs.randint(0, 1 << 32, size=(groups * size + 10, k), dtype=np.uint64).astype(np.uint32)
    for g in range(groups):                                  # member j of group g is row j * groups + g
        rows[g:groups * size:groups, 0:r] = rs.randint(0, 1 << 32, size=r, dtype=np.uint64).astype(np.uint32)
        rows[g:groups * size:groups, r * 3:r * 4] = 17 + g   # a second shared band: the pair matches twice
    ix = be.index(k, b, r, len(rows))
    try:
        for row in rows:
            ix.insert(row[None])
        heads, middle, tails = [(size - 1) * groups + 0], [2 * groups + 1], [0 * groups + 2]
        whole = list(range(3, groups * size, groups))
        alive = np.ones(len(rows), dtype=bool)
        for part in (heads, middle, tails, whole):
            ix.remove(part)
            alive[part] = False
        before = _check(ix, rows, alive, k, b, r, (None, 0.0, 0.5))
        _check_compact(be, ix, rows, alive, k, b, r, before, (None, 0.0, 0.5))
    finally:
        ix.close()


def _collision_rows(rs, k, b, r):
    """Base rows plus members that share a band's fingerprint without sharing its tuple (hash_model second preimages) and
    members whose tuple fingerprints to the tables' empty key (as in test_lsh_self_join.py)."""
    base = rs.randint(0, 1 << 32, size=(120, k), dtype=np.uint64).astype(np.uint32)
    parts = []
    for band in (0, 5, 31):
        sl = slice(band * r, (band + 1) * r)
        for d in rs.permutation(len(base))[:40]:
            t2 = hm.second_preimage(base[d, sl], band, rs)
            if t2 is None:
                continue
            same = base[rs.randint(0, len(base), 3)].copy()
            same[:, sl] = base[d, sl]
            other = base[rs.randint(0, len(base), 3)].copy()
            other[:, sl] = t2
            both = np.empty((6, k), dtype=np.uint32)           # interleaved: colliding tuples alternate along the chain
            both[0::2], both[1::2] = same, other
            parts.append(both)
            break
        else:
            pytest.fail("no second preimage found for band %d" % band)
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, r, rs)
        if e is not None:
            empty = base[rs.randint(0, len(base), 4)].copy()
            empty[:, band * r:(band + 1) * r] = e
            parts.append(empty)
            break
    else:
        pytest.fail("no empty-key tuple found")
    return base, parts


def test_fingerprint_collisions_with_removed_members(be):
    """Chains that mix two tuples with one fingerprint, and the empty-key tuple: remove members between colliding tuples
    (and the chain's head), so the walks pass through removed members to reach the colliding ones behind them."""
    k, b, r = 96, 32, 3
    rs = np.random.RandomState(29)
    base, parts = _collision_rows(rs, k, b, r)
    rows = np.concatenate([base] + parts)
    ix = be.index(k, b, r, len(rows))
    try:
        ix.insert(base)
        for p in parts:
            for row in p:                                     # one at a time: a known chain order
                ix.insert(row[None])
        alive = np.ones(len(rows), dtype=bool)
        start = len(base)
        gone = []
        for p in parts[:3]:
            gone += [start + 1, start + 2, start + 5]         # an 'other', a 'same' and the head of the chain
            start += len(p)
        gone += [start + 1]                                   # one empty-key member
        gone += rs.choice(len(base), 10, replace=False).tolist()
        ix.remove(gone)
        alive[gone] = False
        fp = hm.band_fp(np.concatenate(parts), b, r)
        assert len(np.unique(fp)) < fp.size
        before = _check(ix, rows, alive, k, b, r, (None, 0.0, 0.05))
        _check_compact(be, ix, rows, alive, k, b, r, before, (None, 0.0, 0.05))
    finally:
        ix.close()


def test_remove_insert_tokens_remove_again_compact(be):
    """Remove, then insert more rows through the fused insert_tokens route and plainly, remove again (old and new
    documents), check, compact, insert after the compaction and check again."""
    k, b, r = 128, 32, 4
    rs = np.random.RandomState(41)
    n = 90 if be.name == "emu" else 2000
    lens = rs.randint(1, 120, size=n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    perms = o.init_permutations(k, 5)
    tsig = oc.minhash_bulk_u32tok(tok, off, perms)
    first = tsig[rs.choice(n, n // 3, replace=False)].copy()          # exact duplicates of token documents
    first[::2, :k // 8] = rs.randint(0, 1 << 32, size=(len(first[::2]), k // 8), dtype=np.uint64).astype(np.uint32)
    last = tsig[rs.choice(n, 20, replace=False)].copy()
    ix = be.index(k, b, r, len(first) + n + len(last) + 30)
    try:
        ix.insert(first)
        alive = np.ones(len(first), dtype=bool)
        g1 = rs.choice(len(first), len(first) // 4, replace=False)
        ix.remove(g1)
        alive[g1] = False
        ix.insert_tokens(tok, off, perms)
        ix.insert(last)
        rows = np.concatenate([first, tsig, last])
        alive = np.concatenate([alive, np.ones(n + len(last), dtype=bool)])
        g2 = np.concatenate([rs.choice(np.flatnonzero(alive[:len(first)]), 5, replace=False),
                             len(first) + rs.choice(n + len(last), n // 5, replace=False)])
        ix.remove(g2)
        alive[g2] = False
        before = _check(ix, rows, alive, k, b, r, (None, 0.9))
        _check_compact(be, ix, rows, alive, k, b, r, before, (None, 0.9))
        rows, alive = np.concatenate([rows[alive], tsig[:30]]), np.ones(int(alive.sum()) + 30, dtype=bool)
        ix.insert(tsig[:30])
        _check(ix, rows, alive, k, b, r, (None, 0.9))
    finally:
        ix.close()


def test_capacity_is_given_back_by_compact(be):
    """A full index refuses more rows, also after removals; compact() frees the removed documents' capacity."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(8)
    cap = 64
    rows = _low_entropy(rs, cap, k, 3)
    more = _low_entropy(rs, cap // 2, k, 3)
    ix = be.index(k, b, r, cap)
    try:
        ix.insert(rows)
        assert not ix.try_insert(more[:1])
        gone = rs.choice(cap, cap // 2, replace=False)
        ix.remove(gone)
        assert not ix.try_insert(more[:1])                  # removed numbers are not reused before compact()
        alive = np.ones(cap, dtype=bool)
        alive[gone] = False
        before = _check(ix, rows, alive, k, b, r)
        _check_compact(be, ix, rows, alive, k, b, r, before)
        assert ix.try_insert(more)
        assert not ix.try_insert(more[:1])
        _check(ix, np.concatenate([rows[alive], more]), np.ones(cap, dtype=bool), k, b, r)
    finally:
        ix.close()


def test_empty_one_document_remove_all_and_nothing_removed(be):
    k, b, r = 64, 8, 8
    ix = be.index(k, b, r, 10)
    try:
        assert len(ix.compact()) == 0 and len(ix.alive()) == 0      # empty index
        ix.remove([])
        row = np.arange(k, dtype=np.uint32)[None]
        ix.insert(row)
        assert np.array_equal(ix.compact(), [0])                   # nothing removed: the identity
        ix.remove([0])
        ptr, idx = ix.query(row)
        assert list(ptr) == [0, 0] and len(idx) == 0
        for t in (None, 1.0):
            ptr, idx, eq = ix.pairs(t)
            assert list(ptr) == [0, 0] and len(idx) == 0
            assert ix.clusters(t).tolist() == [-1]
        assert ix.compact().tolist() == [-1]
        assert len(ix.alive()) == 0 and list(ix.pairs()[0]) == [0] and len(ix.clusters()) == 0
        rs = np.random.RandomState(1)
        rows = _low_entropy(rs, 10, k, 2)
        ix.insert(rows)
        assert np.array_equal(ix.compact(), np.arange(10))          # identity again, nothing rebuilt
        _check(ix, rows, np.ones(10, dtype=bool), k, b, r)
        ix.remove(np.arange(10))                                    # remove everything
        before = _check(ix, rows, np.zeros(10, dtype=bool), k, b, r)
        _check_compact(be, ix, rows, np.zeros(10, dtype=bool), k, b, r, before)
    finally:
        ix.close()


def test_c_abi_validation_and_status_counts(emu_lib):
    """Null handle, n < 0, null buffers, a short or misaligned workspace: DSK_ERR_INVALID.  d_status counts ids out of
    range and ids removed already (a repeat within one call included), and a repeated call changes nothing."""
    lib, k = emu_lib, 32
    buf = _aligned(np.zeros(64, dtype=np.int64))
    assert lib.dsk_lsh_remove(None, _p(buf), 1, _p(buf), None) == DSK_ERR_INVALID
    assert b"null handle" in lib.dsk_last_error()
    assert lib.dsk_lsh_alive(None, _p(buf), 1, _p(buf), None) == DSK_ERR_INVALID
    assert b"null handle" in lib.dsk_last_error()
    assert lib.dsk_lsh_compact(None, _p(buf), _p(buf), 512, None) == DSK_ERR_INVALID
    assert b"null handle" in lib.dsk_last_error()
    assert lib.dsk_lsh_compact_workspace_size(None) == 0
    ix = _EmuRmIndex(lib, k, 8, 4, 100)
    try:
        assert lib.dsk_lsh_compact_workspace_size(ix.h) == 0
        assert lib.dsk_lsh_compact(ix.h, None, None, 0, None) == DSK_OK        # empty index: nothing to write
        ix.insert(np.arange(40 * k, dtype=np.uint32).reshape(40, k) % 7)
        for fn in (lib.dsk_lsh_remove, lib.dsk_lsh_alive):
            assert fn(ix.h, _p(buf), -1, _p(buf), None) == DSK_ERR_INVALID
            assert b"n must be" in lib.dsk_last_error()
            for args in ((None, _p(buf)), (_p(buf), None)):
                assert fn(ix.h, args[0], 3, args[1], None) == DSK_ERR_INVALID
                assert b"null buffer" in lib.dsk_last_error()
            assert fn(ix.h, None, 0, None, None) == DSK_OK                     # n = 0: nothing to read or write
        need = lib.dsk_lsh_compact_workspace_size(ix.h)
        assert need > 0
        ws = _aligned(np.zeros(need + 64, dtype=np.uint8))
        remap = np.zeros(40, dtype=np.int32)
        assert lib.dsk_lsh_compact(ix.h, None, _p(ws), need, None) == DSK_ERR_INVALID
        assert lib.dsk_lsh_compact(ix.h, _p(remap), None, need, None) == DSK_ERR_INVALID
        assert b"null buffer" in lib.dsk_last_error()
        assert lib.dsk_lsh_compact(ix.h, _p(remap), _p(ws), need - 1, None) == DSK_ERR_INVALID
        assert b"workspace" in lib.dsk_last_error()
        assert lib.dsk_lsh_compact(ix.h, _p(remap), ctypes.c_void_p(ws.ctypes.data + 4), need, None) == DSK_ERR_INVALID
        assert ix.n == 40 and np.all(ix.alive())                               # nothing happened
        st = ix.remove([3, -1, 40, 2 ** 31 - 1, 5, 3, 7, -(2 ** 31)])
        assert st.tolist() == [4, 1]
        assert ix.remove([3, 5, 7]).tolist() == [0, 3]                         # idempotent: all three removed already
        assert ix.remove([9, 9, 9, 100]).tolist() == [1, 2]
        alive = np.ones(40, dtype=bool)
        alive[[3, 5, 7, 9]] = False
        assert np.array_equal(ix.alive(), alive)
        assert ix.alive([-1, 0, 3, 39, 40, 2 ** 31 - 1]).tolist() == [False, True, False, True, False, False]
        big = _aligned(np.arange(1000, dtype=np.int32) % 41 - 1)              # several warps and CTAs of ids
        status = np.zeros(2, dtype=np.int64)
        assert lib.dsk_lsh_remove(ix.h, _p(big), len(big), _p(status), None) == 0
        # id -1 is out of range; every occurrence of the 4 removed ids, and all but the first occurrence of the 36 others,
        # count as removed already
        occ = np.bincount(np.arange(1000) % 41, minlength=41)
        assert status.tolist() == [int(occ[0]), int(occ[1:].sum()) - 36]
        assert not np.any(ix.alive())
    finally:
        ix.close()


# ---- reference parity (tests/golden/lsh_remove.npz) ---------------------------------------------------------------------
def _golden_lists(g, which):
    ptr, idx = g[which + "_ptr"], g[which + "_idx"]
    return [idx[ptr[i]:ptr[i + 1]].tolist() for i in range(len(ptr) - 1)]


def test_dict_oracle_remove_is_the_reference(golden):
    """_DictLSH.remove restates lsh.py:509-528: its query lists equal the reference's, after the removals and after a few
    removed keys were inserted again."""
    g, sig = golden("lsh_remove"), golden("lsh")["sig"].astype(np.uint64)
    b, r = g["b_r"].tolist()
    ref = _DictLSH(128, b, r)
    for i, row in enumerate(sig):
        ref.insert(i, row)
    for key in g["removed"].tolist():
        ref.remove(key)
    with pytest.raises(ValueError, match="does not exist"):
        ref.remove(int(g["removed"][0]))
    assert [sorted(ref.query(row)) for row in sig] == _golden_lists(g, "query")
    assert all(ref.hashtables[j] for j in range(b)) and all(len(s) for t in ref.hashtables for s in t.values())
    for key in g["reinserted"].tolist():
        ref.insert(key, sig[key])
    assert [sorted(ref.query(row)) for row in sig] == _golden_lists(g, "query2")


def test_golden_query_after_remove_and_reinsert(be, golden):
    """The reference's MinHashLSH.query lists after remove, and after re-inserting removed keys (new document numbers
    that map to the old keys), then after compact() as well."""
    g, sig = golden("lsh_remove"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    removed, back = g["removed"].tolist(), g["reinserted"].tolist()
    ix = be.index(128, b, r, len(sig) + len(back))
    try:
        ix.insert(sig)
        ix.remove(removed)
        keys = list(range(len(sig)))

        def lists():
            ptr, idx = ix.query(sig)
            return [sorted(keys[d] for d in idx[ptr[q]:ptr[q + 1]].tolist()) for q in range(len(sig))]

        assert lists() == _golden_lists(g, "query")
        ix.insert(sig[back])
        keys += back
        assert lists() == _golden_lists(g, "query2")
        remap = ix.compact()
        keys = [kk for kk, m in zip(keys, remap) if m >= 0]
        assert lists() == _golden_lists(g, "query2")
    finally:
        ix.close()


def test_thread_sanitizer_removal_aware_clusters():
    """Both cluster paths of the removal-aware kernels under ThreadSanitizer (tests/emu/emu_tsan_remove_main.cpp): one
    big component with removed members hooked by hundreds of host threads at once; the labels are also checked against a
    serial union-find of the remaining documents' brute-force pairs."""
    out = os.path.join(EMU, "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "emu_tsan_remove")
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-ffp-contract=off", "-fsanitize=thread", "-DDSK_EMU",
                            "-I" + EMU, "-o", exe, os.path.join(EMU, "emu_capi.cpp"),
                            os.path.join(EMU, "emu_tsan_remove_main.cpp")], capture_output=True, text=True)
    if build.returncode != 0:
        pytest.skip("ThreadSanitizer runtime not available: " + build.stderr[-200:])
    env = dict(os.environ, TSAN_OPTIONS="history_size=7 halt_on_error=1 exitcode=66")   # history: see emu_tsan_main.cpp
    run = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=900)
    text = run.stdout + run.stderr
    if run.returncode not in (0, 1, 66) or "unexpected memory mapping" in text:
        pytest.skip("ThreadSanitizer cannot run in this container: " + text[-200:])
    assert "data race" not in text and run.returncode == 0, text[-2000:]
    assert text.count("identical") == 4, text[-2000:]


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_errors_leave_the_index_unchanged():
    """remove() raises the reference's ValueError for an id out of range, removed already or listed twice -- before it
    changes anything; it takes one number, a list, a numpy array or a CUDA tensor."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(2)
    k = 64
    rows = _low_entropy(rs, 200, k, 3)
    ix = dsk.GpuLSH(num_perm=k, params=(16, 4), capacity=300)
    ix.insert(rows, keys=["k%d" % i for i in range(200)])
    ix.remove(5)
    ix.remove([6, 7])
    ix.remove(np.array([8, 9], dtype=np.uint16))
    ix.remove(torch.tensor([10, 11], device="cuda"))
    alive = np.ones(200, dtype=bool)
    alive[5:12] = False
    snapshot = (_pairs_dict(*ix.candidate_pairs()), ix.duplicate_clusters().tolist(), ix.alive().tolist())
    assert snapshot[2] == alive.tolist()
    for bad in (200, -1, [1, 2, 300], [5], [1, 12, 7], [3, 3], np.array([4, 13, 4]), torch.tensor([2 ** 40], device="cuda")):
        with pytest.raises(ValueError, match="The given key does not exist"):
            ix.remove(bad)
        assert (_pairs_dict(*ix.candidate_pairs()), ix.duplicate_clusters().tolist(), ix.alive().tolist()) == snapshot
    with pytest.raises(TypeError):
        ix.remove([1.5])
    assert ix.alive([0, 5, 199, 200, -3]).tolist() == [True, False, True, False, False]
    m = ix.alive(to_host=False)
    assert m.is_cuda and m.dtype == torch.bool and len(ix) == 200
    remap = ix.compact(to_host=False)
    assert remap.is_cuda and remap.dtype == torch.int32 and len(ix) == 193
    assert ix.keys == ["k%d" % i for i in range(200) if alive[i]]
    assert ix.query_keys(rows[12:13])[0].count("k12") == 1


@pytest.mark.gpu
def test_c3_scale_remove_duplicates_one_million_documents():
    """The C3 workload at 1M documents (128 tokens, K = 256, LSH(0.8), 10 % planted near-duplicates) built through
    insert_tokens.  Remove the non-root members of duplicate_clusters(0.8) and a random 5 % more: the pairs equal the
    earlier pairs among the remaining documents, the labels equal scipy's components of them, and after compact() both
    map through remap."""
    import torch
    import datasketch_b200 as dsk
    from datasketch_b200.minhash import _make_permutations
    n, t, k = 1_000_000, 128, 256
    perms = _make_permutations(k, 1)
    g = torch.Generator(device="cuda").manual_seed(3)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, t), dtype=torch.int32, device="cuda", generator=g)
    ndup = n // 10
    src = torch.randint(0, n, (ndup,), device="cuda", generator=g)
    dst = torch.randint(0, n, (ndup,), device="cuda", generator=g)
    tok[dst] = tok[src]
    mask = torch.rand((ndup, t), device="cuda", generator=g) < 0.1
    tok[dst] = torch.where(mask, torch.randint(-2 ** 31, 2 ** 31 - 1, (ndup, t), dtype=torch.int32, device="cuda", generator=g),
                           tok[dst])
    off = torch.arange(0, (n + 1) * t, t, dtype=torch.int64, device="cuda")
    ix = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=n)
    ix.insert_tokens(tok.view(-1), off, n * t, perms)
    before = {thr: ix.candidate_pairs(thr) for thr in (None, 0.8)}
    labels = ix.duplicate_clusters(0.8)
    rs = np.random.RandomState(0)
    gone = np.flatnonzero(labels != np.arange(n))
    assert len(gone) > ndup // 4
    extra = rs.choice(np.flatnonzero(labels == np.arange(n)), n // 20, replace=False)
    gone = np.concatenate([gone, extra])
    ix.remove(torch.from_numpy(gone).cuda())
    alive = np.ones(n, dtype=bool)
    alive[gone] = False
    assert np.array_equal(ix.alive(), alive)
    remap = None
    for stage in ("removed", "compacted"):
        for thr in (None, 0.8):
            ptr0, idx0, eq0 = before[thr]
            rows0 = np.repeat(np.arange(n), np.diff(ptr0))
            keep = alive[rows0] & alive[idx0]
            ptr, idx, eq = ix.candidate_pairs(thr)
            got_rows = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
            if stage == "removed":
                want_rows, want_idx = rows0[keep], idx0[keep].astype(np.int64)
            else:
                want_rows, want_idx = remap[rows0[keep]], remap[idx0[keep]]
            w = np.lexsort((want_idx, want_rows))
            gsort = np.lexsort((idx, got_rows))
            assert np.array_equal(got_rows[gsort], want_rows[w]) and np.array_equal(idx[gsort], want_idx[w])
            assert np.array_equal(eq[gsort], eq0[keep][w])
            lab = ix.duplicate_clusters(thr).astype(np.int64)
            m = len(ptr) - 1
            comp = _components(m, zip(got_rows.tolist(), idx.tolist()))
            if stage == "removed":
                comp[~alive] = -1
            assert np.array_equal(lab, comp), (stage, thr)
        if stage == "removed":
            labels_removed = ix.duplicate_clusters().astype(np.int64)
            remap = ix.compact().astype(np.int64)
            assert np.array_equal(remap, np.where(alive, np.cumsum(alive) - 1, -1)) and len(ix) == int(alive.sum())
            assert np.array_equal(ix.duplicate_clusters(), remap[labels_removed[alive]])
