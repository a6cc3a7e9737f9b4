"""GpuLSH.query_jaccard / query_best: query rows that are not in the index, verified on the device.

``query_jaccard(sig, min_jaccard)`` lists, per query row, each candidate of ``query`` once with ``eq``, the number of the K
positions where the query row and the document's row agree (eq / K is MinHash.jaccard, minhash.py:324), keeping those with
MinHash.jaccard >= min_jaccard -- ``[d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]`` (lsh.py:370-432).
``query_best`` gives each query's kept candidate with the largest eq, the smallest document among equal ones, or -1 / -1.

The oracle is the dict-bucket index oracle_np.DictLSH.query (with test_lsh_remove.py's MinHashLSH.remove), oracle_np.jaccard
and a max with that tie-break; tests/golden/lsh_query_jaccard.npz (oracle/gen_golden_lsh_query_jaccard.py) pins it to the
reference.  The two backends are those of test_lsh_self_join.py: ``emu``, the whole library on the emulation shim driven
through its C-ABI, and ``gpu``, the Python API on the H100.
"""
import os
import sys

import numpy as np
import pytest

from oracle import oracle_clib as oc
from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402
from test_lsh_self_join import _aligned, _low_entropy, _min_count, _p, _pairs_dict  # noqa: E402
from test_lsh_remove import _EmuRmIndex, _GpuRmIndex, _csr_sets, _oracle_index  # noqa: E402

DSK_OK, DSK_ERR_INVALID = 0, 1


# ---- backends ----------------------------------------------------------------------------------------------------------
class _EmuQIndex(_EmuRmIndex):
    """The emulated library through its C-ABI, with the query-verify entries."""

    def query_jaccard(self, sig, min_jaccard=None):
        lib, sig, mc = self.lib, _aligned(np.asarray(sig, dtype=np.uint32)), _min_count(min_jaccard, self.k)
        nq = len(sig)
        counts, ptr = np.full(nq + 1, -7, dtype=np.int64), np.zeros(nq + 1, dtype=np.int64)
        scratch = np.zeros(nq // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_query_jaccard_count(self.h, _p(sig), nq, mc, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), nq, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        idx, eq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_query_jaccard_fill(self.h, _p(sig), nq, mc, _p(ptr), _p(idx), _p(eq), None) == 0, \
            lib.dsk_last_error()
        return ptr, idx[:m], eq[:m]

    def query_best(self, sig, min_jaccard=None):
        lib, sig, mc = self.lib, _aligned(np.asarray(sig, dtype=np.uint32)), _min_count(min_jaccard, self.k)
        nq = len(sig)
        idx, eq = np.full(max(nq, 1), -7, dtype=np.int32), np.full(max(nq, 1), -7, dtype=np.int32)
        assert lib.dsk_lsh_query_best(self.h, _p(sig), nq, mc, _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return idx[:nq], eq[:nq]


class _Emu:
    name = "emu"
    grid_rows = 2 * 8 * 8          # two emulated SMs x 8 CTAs x 8 warps: queries one sweep of the walk covers

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuQIndex(self.lib, k, b, r, capacity)


class _GpuQIndex(_GpuRmIndex):
    def query_jaccard(self, sig, min_jaccard=None):
        return self.ix.query_jaccard(np.ascontiguousarray(sig, dtype=np.uint32), min_jaccard)

    def query_best(self, sig, min_jaccard=None):
        return self.ix.query_best(np.ascontiguousarray(sig, dtype=np.uint32), min_jaccard)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk
        self.grid_rows = dsk._native.device_info(0)["sm_count"] * 8 * 8

    def index(self, k, b, r, capacity):
        return _GpuQIndex(self.dsk, k, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
def _want(ref, rows, qsig, min_jaccard):
    """Per query {d: eq} over DictLSH.query(query row) with oracle_np.jaccard >= min_jaccard (None: all)."""
    rows, qsig = np.asarray(rows, dtype=np.uint64), np.asarray(qsig, dtype=np.uint64)
    out = []
    for q in qsig:
        out.append({d: int(np.count_nonzero(q == rows[d])) for d in ref.query(q)
                    if min_jaccard is None or o.jaccard(q, rows[d]) >= min_jaccard})
    return out


def _best(want):
    """Per query (d, eq) of the largest eq, the smallest d among equal ones; (-1, -1) for none."""
    return [min(((-e, d) for d, e in w.items()), default=(1, -1)) for w in want]


def _got(ptr, idx, eq):
    """CSR result -> per query {d: eq}; each candidate listed once."""
    assert ptr[0] == 0 and np.all(np.diff(ptr) >= 0) and ptr[-1] == len(idx) == len(eq)
    out = []
    for q in range(len(ptr) - 1):
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        d = dict(zip(idx[sl].tolist(), eq[sl].tolist()))
        assert len(d) == ptr[q + 1] - ptr[q], q
        out.append(d)
    return out


def _check(ix, rows, qsig, k, b, r, thresholds, alive=None):
    """query_jaccard and query_best of qsig against the oracle over rows (removed ones excluded), per threshold; the
    unfiltered candidates equal query()'s."""
    rows = np.asarray(rows, dtype=np.uint32)
    alive = np.ones(len(rows), dtype=bool) if alive is None else alive
    ref = _oracle_index(rows, alive, k, b, r)
    for t in thresholds:
        want = _want(ref, rows, qsig, t)
        got = _got(*ix.query_jaccard(qsig, t))
        assert got == want, t
        bi, be_ = ix.query_best(qsig, t)
        assert [(-int(e), int(d)) if d >= 0 else (1, -1) for d, e in zip(bi, be_)] == [
            (e, d) if d >= 0 else (1, -1) for e, d in _best(want)], t
        assert all((d >= 0) == (e >= 0) for d, e in zip(bi.tolist(), be_.tolist()))
        if t is None:
            assert [set(w) for w in got] == _csr_sets(*ix.query(qsig))
    return ref


def _perturb(rs, rows, frac, vals):
    out = np.array(rows, dtype=np.uint32, copy=True)
    m = rs.rand(*out.shape) < frac
    out[m] = rs.randint(0, vals, size=int(m.sum())).astype(np.uint32)
    return out


# ---- cases -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,b,r,vals", [(32, 8, 4, 3), (100, 33, 3, 4)])
def test_low_entropy_mixed_queries(be, k, b, r, vals):
    """Big buckets and (for b = 33) two lane rounds; queries mix indexed rows, perturbed rows and unrelated rows.
    Thresholds: none, 0.0, 1.0 and the exact boundaries c / K and (c + 1) / K."""
    rs = np.random.RandomState(k + b)
    n = (150 if b <= 32 else 90) if be.name == "emu" else 2500
    nq = 60 if be.name == "emu" else 1500
    sig = _low_entropy(rs, n, k, vals)
    third = nq // 3
    qsig = np.concatenate([sig[rs.choice(n, third)], _perturb(rs, sig[rs.choice(n, third)], 0.1, vals),
                           _low_entropy(rs, nq - 2 * third, k, vals)])
    ix = be.index(k, b, r, n)
    ix.insert(sig[:n // 2])
    ix.insert(sig[n // 2:])
    try:
        c = k // 3
        _check(ix, sig, qsig, k, b, r, (None, 0.0, 1.0, c / k, (c + 1) / k))
    finally:
        ix.close()


def test_queries_equal_to_the_index_rows(be):
    """Querying the index with its own rows: the candidates are query()'s; restricted to d < i they are candidate_pairs'
    with the same eq; every row finds itself with eq = K and query_best returns it (the smallest of its exact copies)."""
    k, b, r, vals = 64, 16, 4, 3
    rs = np.random.RandomState(11)
    n = 140 if be.name == "emu" else 3000
    sig = _low_entropy(rs, n, k, vals)
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        for t in (None, 0.5):
            got = _got(*ix.query_jaccard(sig, t))
            pairs = _pairs_dict(*ix.pairs(t))
            assert {(i, d): e for i, g in enumerate(got) for d, e in g.items() if d < i} == pairs, t
            assert all(g.get(i) == k for i, g in enumerate(got))
            bi, bq = ix.query_best(sig, t)
            first = {}
            for i, row in enumerate(sig):
                first.setdefault(row.tobytes(), i)
            assert bi.tolist() == [first[row.tobytes()] for row in sig] and np.all(bq == k)
        assert [set(g) for g in _got(*ix.query_jaccard(sig))] == _csr_sets(*ix.query(sig))
    finally:
        ix.close()


@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_are_no_candidates(be, head_collides):
    """Indexed tuples that share a band's fingerprint without being equal (hash_model second preimages, in bands 0, 31
    and 35 -- the second lane round) and the tuple whose fingerprint is the tables' empty key.  A query carrying one tuple
    of a colliding pair meets the members with the other tuple in its chain and must skip them, also when the chain's
    head (its last inserted member) is one of them."""
    k, b, r = 120, 40, 3
    rs = np.random.RandomState(31 + head_collides)
    base = rs.randint(0, 1 << 32, size=(100, k), dtype=np.uint64).astype(np.uint32)
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
            q = rs.randint(0, 1 << 32, size=(2, k), dtype=np.uint64).astype(np.uint32)   # fresh rows with one tuple each
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
        ref = _check(ix, rows, qsig, k, b, r, (None, 0.0, 0.05))
        want = _want(ref, rows, qsig, None)
        for j in range(3):                                            # each colliding query meets only its own tuple's rows
            assert len(want[2 * j]) == 3 and len(want[2 * j + 1]) == 2
        assert len(want[6]) == 3                                      # the empty-key tuple's members
    finally:
        ix.close()


def test_removed_documents_are_never_returned(be):
    """Removed chain heads, middles and tails (and a whole bucket): query_jaccard skips them and query_best never picks
    one, before compact() and, through remap, after it."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(3)
    groups, size = 4, 5
    rows = rs.randint(0, 1 << 32, size=(groups * size + 10, k), dtype=np.uint64).astype(np.uint32)
    for g in range(groups):                                      # member j of group g is row j * groups + g
        rows[g:groups * size:groups, 0:r] = rs.randint(0, 1 << 32, size=r, dtype=np.uint64).astype(np.uint32)
        rows[g:groups * size:groups, r * 3:r * 4] = 17 + g
    qsig = np.concatenate([rows, _perturb(rs, rows, 0.2, 1 << 30)])
    qsig[len(rows):, 0:r] = rows[:, 0:r]                         # the perturbed copies keep their first band
    ix = be.index(k, b, r, len(rows))
    try:
        for row in rows:
            ix.insert(row[None])
        alive = np.ones(len(rows), dtype=bool)
        for part in ([(size - 1) * groups + 0], [2 * groups + 1], [0 * groups + 2], list(range(3, groups * size, groups))):
            ix.remove(part)
            alive[part] = False
        thresholds = (None, 0.0, 0.5)
        _check(ix, rows, qsig, k, b, r, thresholds, alive)
        before = {t: _got(*ix.query_jaccard(qsig, t)) for t in thresholds}
        bi, _ = ix.query_best(qsig)
        assert np.all(alive[bi[bi >= 0]])
        remap = np.asarray(ix.compact(), dtype=np.int64)
        _check(ix, rows[alive], qsig, k, b, r, thresholds)
        for t in thresholds:
            assert _got(*ix.query_jaccard(qsig, t)) == [{int(remap[d]): e for d, e in g.items()} for g in before[t]]
    finally:
        ix.close()


def test_rows_from_the_fused_token_insert(be):
    """Documents inserted from tokens (the signature kernel's fused insert epilogue) between plain inserts; the queries
    are near-duplicate documents of them, and removals happen in between."""
    k, b, r = 128, 32, 4
    rs = np.random.RandomState(5)
    n = 100 if be.name == "emu" else 3000
    lens = rs.randint(1, 200, size=n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    perms = o.init_permutations(k, 5)
    sig = oc.minhash_bulk_u32tok(tok, off, perms)
    qtok = tok.copy()
    qtok[rs.rand(len(qtok)) < 0.1] = rs.randint(0, 1 << 32, dtype=np.uint64)   # 10 % of the tokens resampled
    qsig = np.concatenate([oc.minhash_bulk_u32tok(qtok, off, perms),
                           rs.randint(0, 1 << 32, size=(10, k), dtype=np.uint64).astype(np.uint32)])
    before = rs.randint(0, 1 << 32, size=(20, k), dtype=np.uint64).astype(np.uint32)
    ix = be.index(k, b, r, n + 40)
    try:
        ix.insert(before)
        ix.insert_tokens(tok, off, perms)
        ix.insert(sig[:20])
        rows = np.concatenate([before, sig, sig[:20]])
        ref = _check(ix, rows, qsig, k, b, r, (None, 0.7, 0.9))
        assert sum(len(w) for w in _want(ref, rows, qsig, 0.7)) >= n // 4       # the near-duplicates meet
        alive = np.ones(len(rows), dtype=bool)
        gone = rs.choice(len(rows), len(rows) // 5, replace=False)
        ix.remove(gone)
        alive[gone] = False
        _check(ix, rows, qsig, k, b, r, (None, 0.7), alive)
    finally:
        ix.close()


def test_query_best_ties_go_to_the_smallest_document(be):
    """Several documents share the top eq with a query, found through different bands (different lanes) and through one
    band (one lane's chain, walked from the last inserted): the smallest document number wins.  A unique better one wins
    over them; -1 / -1 when nothing matches or the filter keeps nothing."""
    k, b, r = 64, 16, 4
    rs = np.random.RandomState(77)
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
    docs = []
    for j in range(6):                                           # eq = K - 8: bands 0..j-1 broken, band j intact
        for _ in range(2):                                       # two per band: the same lane's chain
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
    rows = rows[order]                                           # document numbers in shuffled order
    ties = [i for i in range(len(rows)) if len(noise) <= order[i] < len(noise) + 12]
    assert all(np.count_nonzero(rows[i] == q) == k - 8 for i in ties)
    better = q.copy()
    better[[b * r - 1]] += 1                                     # eq = K - 1
    far = rs.randint(0, 1 << 32, size=(1, k), dtype=np.uint64).astype(np.uint32)
    qsig = np.stack([q, q, far[0]])
    ix = be.index(k, b, r, len(rows) + 1)
    try:
        for row in rows:
            ix.insert(row[None])
        bi, bq = ix.query_best(qsig[:1])
        assert bi.tolist() == [ties[0]] and bq.tolist() == [k - 8]
        _check(ix, rows, qsig, k, b, r, (None, (k - 8) / k, (k - 7) / k, 1.0))
        bi, bq = ix.query_best(qsig, (k - 7) / k)                 # the filter keeps nothing
        assert bi.tolist() == [-1, -1, -1] and bq.tolist() == [-1, -1, -1]
        bi, bq = ix.query_best(far)                              # nothing matches
        assert bi.tolist() == [-1] and bq.tolist() == [-1]
        ix.insert(better[None])                                  # the largest number, but the best eq
        bi, bq = ix.query_best(q[None])
        assert bi.tolist() == [len(rows)] and bq.tolist() == [k - 1]
    finally:
        ix.close()


def test_empty_one_document_and_no_queries(be):
    k, b, r = 64, 8, 8
    ix = be.index(k, b, r, 10)
    row = np.arange(k, dtype=np.uint32)[None]
    try:
        ptr, idx, eq = ix.query_jaccard(row)                       # empty index
        assert list(ptr) == [0, 0] and len(idx) == 0 and len(eq) == 0
        assert [x.tolist() for x in ix.query_best(row)] == [[-1], [-1]]
        ix.insert(row)
        for t in (None, 0.0, 1.0):
            assert _got(*ix.query_jaccard(row, t)) == [{0: k}]
            assert [x.tolist() for x in ix.query_best(row, t)] == [[0], [k]]
        near = row.copy()
        near[0, 0] += 1
        assert _got(*ix.query_jaccard(near)) == [{0: k - 1}] and _got(*ix.query_jaccard(near, 1.0)) == [{}]
        ptr, idx, eq = ix.query_jaccard(np.zeros((0, k), dtype=np.uint32))    # no queries
        assert list(ptr) == [0] and len(idx) == 0
        assert [len(x) for x in ix.query_best(np.zeros((0, k), dtype=np.uint32))] == [0, 0]
    finally:
        ix.close()


def test_more_queries_than_one_grid_sweep(be):
    """Queries beyond one sweep of the grid: the walk's grid-stride loop over queries."""
    k, b, r = 32, 8, 4
    rs = np.random.RandomState(9)
    n = 200 if be.name == "emu" else 5000
    sig = _low_entropy(rs, n, k, 4)
    nq = 3 * be.grid_rows + 5
    qsig = _perturb(rs, sig[rs.randint(0, n, nq)], 0.1, 4)
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        _check(ix, sig, qsig, k, b, r, (None, 0.6))
    finally:
        ix.close()


@pytest.mark.parametrize("k", [2048, 4096])
def test_large_k_fewer_warps_per_cta(be, k):
    """K = 2048 (4 warps per CTA) and K = 4096 (2 warps): each warp's row still fits the shared memory it is given."""
    b, r = 16, 4
    rs = np.random.RandomState(k)
    n = 40
    sig = rs.randint(0, 4, size=(n, k)).astype(np.uint32)
    sig[:, b * r:] = rs.randint(0, 1 << 32, size=(n, k - b * r), dtype=np.uint64).astype(np.uint32)
    sig[10:20] = sig[0:10]
    sig[20:25, b * r:] = sig[0:5, b * r:]
    qsig = np.concatenate([sig[:12], _perturb(rs, sig[12:30], 0.3, 4)])
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        _check(ix, sig, qsig, k, b, r, (None, 0.5, 0.99))
    finally:
        ix.close()


def test_c_abi_argument_validation(emu_lib):
    """Null handle, nq < 0, min_count outside [0, K], null buffers with nq > 0: DSK_ERR_INVALID.  nq == 0 with null
    buffers is a valid no-op."""
    lib, k = emu_lib, 32
    buf = _aligned(np.zeros(256, dtype=np.int64))
    entries = ((lib.dsk_lsh_query_jaccard_count, 1), (lib.dsk_lsh_query_jaccard_fill, 3), (lib.dsk_lsh_query_best, 2))
    for fn, nb in entries:
        assert fn(None, _p(buf), 1, 0, *[_p(buf)] * nb, None) == DSK_ERR_INVALID
        assert b"null handle" in lib.dsk_last_error()
    ix = _EmuQIndex(lib, k, 8, 4, 20)
    try:
        ix.insert(np.arange(3 * k, dtype=np.uint32).reshape(3, k) % 5)
        for fn, nb in entries:
            assert fn(ix.h, _p(buf), -1, 0, *[_p(buf)] * nb, None) == DSK_ERR_INVALID
            assert b"nq must be" in lib.dsk_last_error()
            for mc in (-1, k + 1, -(1 << 31)):
                assert fn(ix.h, _p(buf), 1, mc, *[_p(buf)] * nb, None) == DSK_ERR_INVALID
                assert b"min_count" in lib.dsk_last_error()
            assert fn(ix.h, None, 1, 0, *[_p(buf)] * nb, None) == DSK_ERR_INVALID        # no query matrix
            assert b"null buffer" in lib.dsk_last_error()
            for j in range(nb):                                                          # any one null output buffer
                args = [_p(buf)] * nb
                args[j] = None
                assert fn(ix.h, _p(buf), 1, 0, *args, None) == DSK_ERR_INVALID
                assert b"null buffer" in lib.dsk_last_error()
            assert fn(ix.h, None, 0, 0, *[None] * nb, None) == DSK_OK                   # nq = 0: nothing to read or write
            assert fn(ix.h, _p(buf), 1, k, *[_p(buf)] * nb, None) == DSK_OK
    finally:
        ix.close()


# ---- reference parity (tests/golden/lsh_query_jaccard.npz) ----------------------------------------------------------------
def _golden_lists(g, which):
    ptr, idx = g[which + "_ptr"], g[which + "_idx"]
    return [idx[ptr[i]:ptr[i + 1]].tolist() for i in range(len(ptr) - 1)]


def test_oracle_is_the_reference(golden):
    """DictLSH.query + oracle_np.jaccard give the reference's MinHashLSH.query lists, MinHash.jaccard values and filtered
    lists for held-out queries against lsh.npz's 300 documents."""
    g, sig = golden("lsh_query_jaccard"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    ref = _oracle_index(sig, np.ones(len(sig), dtype=bool), 128, b, r)
    qsig = g["qsig"].astype(np.uint64)
    assert [sorted(ref.query(q)) for q in qsig] == _golden_lists(g, "query")
    jac = [o.jaccard(q, sig[d].astype(np.uint64)) for q, lst in zip(qsig, _golden_lists(g, "query")) for d in lst]
    assert jac == g["query_jaccard"].tolist()
    for j, t in enumerate(g["thresholds"].tolist()):
        assert [sorted(w) for w in _want(ref, sig, qsig, t)] == _golden_lists(g, "kept%d" % j)
    assert sum(len(x) for x in _golden_lists(g, "kept1")) > 0 and any(len(x) == 0 for x in _golden_lists(g, "query"))


def test_golden_query_jaccard(be, golden):
    """The library gives the reference's candidate lists, MinHash.jaccard * K as eq, the filtered lists, and query_best
    their argmax."""
    g, sig = golden("lsh_query_jaccard"), golden("lsh")["sig"]
    b, r = g["b_r"].tolist()
    qsig = g["qsig"]
    ix = be.index(128, b, r, len(sig))
    try:
        ix.insert(sig)
        got = _got(*ix.query_jaccard(qsig))
        assert [sorted(x) for x in got] == _golden_lists(g, "query")
        assert [x[d] / 128.0 for x in got for d in sorted(x)] == g["query_jaccard"].tolist()
        for j, t in enumerate(g["thresholds"].tolist()):
            kept = _got(*ix.query_jaccard(qsig, t))
            assert [sorted(x) for x in kept] == _golden_lists(g, "kept%d" % j)
            bi, bq = ix.query_best(qsig, t)
            assert list(zip(bi.tolist(), bq.tolist())) == [(d, -e) if d >= 0 else (-1, -1)
                                                           for e, d in _best(kept)]
    finally:
        ix.close()


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_api_errors_and_outputs():
    """Wrong K and non-32-bit tensors raise as query() does; to_host=False returns CUDA tensors; query() is unchanged."""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(4)
    k = 64
    rows = _low_entropy(rs, 300, k, 3)
    ix = dsk.GpuLSH(num_perm=k, params=(16, 4), capacity=300)
    ix.insert(rows)
    q = _perturb(rs, rows[:50], 0.1, 3)
    p0, i0 = ix.query(q)
    for fn in (ix.query, ix.query_jaccard, ix.query_best):
        with pytest.raises(ValueError, match="Expecting minhash with length"):
            fn(np.zeros((2, k + 1), dtype=np.uint32))
        with pytest.raises(TypeError):
            fn(torch.zeros((2, k), dtype=torch.int64, device="cuda"))
    for fn in (ix.query_jaccard, ix.query_best):
        with pytest.raises(ValueError):
            fn(q, 1.5)
    ptr, idx, eq = ix.query_jaccard(q, 0.3, to_host=False)
    assert ptr.is_cuda and ptr.dtype == torch.int64 and idx.dtype == torch.int32 and eq.dtype == torch.int32
    bi, bq = ix.query_best(torch.from_numpy(q.view(np.int32)).cuda(), 0.3, to_host=False)
    assert bi.is_cuda and bi.dtype == torch.int32 and bq.dtype == torch.int32 and len(bi) == 50
    p1, i1 = ix.query(q)
    assert np.array_equal(p0, p1) and np.array_equal(i0, i1)
    assert [set(x) for x in _got(*ix.query_jaccard(q))] == _csr_sets(p0, i0)


@pytest.mark.gpu
def test_c3_scale_one_million_documents_100k_queries():
    """The C3 workload at 1M documents (128 tokens, K = 256, LSH(0.8)) built through insert_tokens, and 100k fresh
    queries, half of them copies of indexed documents with 10 % of the tokens resampled: query_jaccard and query_best
    equal the two-step flow (query, then codec.jaccard_pairs on the concatenated rows, then the filter and the argmax)."""
    import torch
    import datasketch_b200 as dsk
    from datasketch_b200.minhash import _make_permutations
    n, t, k, nq = 1_000_000, 128, 256, 100_000
    perms = _make_permutations(k, 1)
    g = torch.Generator(device="cuda").manual_seed(5)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, t), dtype=torch.int32, device="cuda", generator=g)
    off = torch.arange(0, (n + 1) * t, t, dtype=torch.int64, device="cuda")
    ix = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=n)
    ix.insert_tokens(tok.view(-1), off, n * t, perms)
    qtok = torch.randint(-2 ** 31, 2 ** 31 - 1, (nq, t), dtype=torch.int32, device="cuda", generator=g)
    src = torch.randint(0, n, (nq // 2,), device="cuda", generator=g)
    mask = torch.rand((nq // 2, t), device="cuda", generator=g) < 0.1
    qtok[:nq // 2] = torch.where(mask, qtok[:nq // 2], tok[src])
    qoff = torch.arange(0, (nq + 1) * t, t, dtype=torch.int64, device="cuda")
    qsig = dsk.engine.bulk_signatures_device(qtok.view(-1), qoff, nq * t, perms)
    sig = dsk.engine.bulk_signatures_device(tok.view(-1), off, n * t, perms)
    qp, qi = ix.query(qsig, to_host=False)
    rows_q = torch.repeat_interleave(torch.arange(nq, device="cuda"), qp[1:] - qp[:-1])
    jac = dsk.codec.jaccard_pairs(torch.cat([sig, qsig]), n + rows_q, qi.long())   # MinHash.jaccard per pair
    cnt = np.rint(jac * k).astype(np.int64)
    rows_q, qi = rows_q.cpu().numpy(), qi.cpu().numpy().astype(np.int64)
    for thr in (None, 0.8):
        keep = np.ones(len(jac), dtype=bool) if thr is None else jac >= thr
        want = np.stack([rows_q[keep], qi[keep], cnt[keep]], 1)
        ptr, idx, eq = ix.query_jaccard(qsig, thr)
        got_rows = np.repeat(np.arange(nq), np.diff(ptr))
        got = np.stack([got_rows, idx.astype(np.int64), eq.astype(np.int64)], 1)
        assert len(got) == len(want) and (thr is not None or len(got) >= nq // 4)
        assert np.array_equal(got[np.lexsort(got.T[::-1])], want[np.lexsort(want.T[::-1])]), thr
        bi, bq = ix.query_best(qsig, thr)
        w_eq = np.full(nq, -1, dtype=np.int64)
        np.maximum.at(w_eq, want[:, 0], want[:, 2])
        w_idx = np.full(nq, np.iinfo(np.int64).max, dtype=np.int64)
        top = want[want[:, 2] == w_eq[want[:, 0]]]
        np.minimum.at(w_idx, top[:, 0], top[:, 1])
        w_idx[w_eq < 0] = -1
        assert np.array_equal(bq, w_eq) and np.array_equal(bi, w_idx), thr
