"""The LSH index and the Jaccard top-k on inputs built to hit their hash collisions and their shared-memory limits.

Both promise exactly the reference's results but find them through a hash:

* GpuLSH buckets each band's r-tuple by a 64-bit fingerprint in an open-addressed table.  Different tuples with one
  fingerprint share a chain and are told apart by comparing the tuples (also when a document that matched an earlier
  band is skipped), and a fingerprint equal to the table's empty key is remapped.
* The top-k prefilter bounds a pair's count of equal positions by the agreement of 16-bit value fingerprints and counts
  exactly only the pairs whose bound could still enter a query's list.

Random signatures practically never collide, so these cases are built from the model of the hashes in
tests/hash_model.py: second preimages of the band fingerprint, a tuple whose fingerprint is the empty key, probe
clusters that wrap past the end of a table, fingerprint twins of top-k values.  Each case first checks that its
collisions really collide in the library, then compares with the dict-bucket oracle (oracle_np.DictLSH, the
reference's lsh.py:326-347, :370-432) or a brute-force ranking (MinHash.jaccard, minhash.py:324).

Every case runs on two backends: ``emu``, the whole library compiled with g++ on the emulation shim
(tests/emu/emu_capi.cpp) and driven through its C-ABI with host buffers, and ``gpu``, the compiled library on the H100
through the Python API.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

from oracle import oracle_clib as oc
from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402


# ---- backends ----------------------------------------------------------------------------------------------------------
def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _aligned(a):
    """A 16-byte aligned copy of ``a`` (device buffers are; the library checks), with slack behind it."""
    a = np.ascontiguousarray(a)
    buf = np.zeros(a.nbytes + 64, dtype=np.uint8)
    s = (-buf.ctypes.data) % 16
    out = buf[s:s + a.nbytes].view(a.dtype).reshape(a.shape)
    out[...] = a
    return out


class _EmuIndex:
    def __init__(self, lib, k, b, r, capacity):
        self.lib, self.k = lib, k
        self.h = ctypes.c_void_p()
        assert lib.dsk_lsh_create(k, b, r, capacity, 0, ctypes.byref(self.h)) == 0, lib.dsk_last_error()

    def insert(self, sig):
        sig = _aligned(np.asarray(sig, dtype=np.uint32))
        assert self.lib.dsk_lsh_insert(self.h, _p(sig), len(sig), None) == 0, self.lib.dsk_last_error()

    def insert_tokens(self, tok, off, perms):
        lib, ph = self.lib, ctypes.c_void_p()
        a, b = np.ascontiguousarray(perms[0]), np.ascontiguousarray(perms[1])
        assert lib.dsk_perm_create(_p(a), _p(b), self.k, 0, ctypes.byref(ph)) == 0, lib.dsk_last_error()
        tok, off = _aligned(tok), _aligned(off)
        rc = lib.dsk_lsh_insert_tokens(self.h, ph, _p(tok), 0, _p(off), len(off) - 1, len(tok), None)
        lib.dsk_perm_destroy(ph)
        assert rc == 0, lib.dsk_last_error()

    def query(self, q):
        lib = self.lib
        q = _aligned(np.asarray(q, dtype=np.uint32))
        nq = len(q)
        counts, ptr = np.zeros(nq + 1, dtype=np.int64), np.zeros(nq + 1, dtype=np.int64)
        scratch = np.zeros(nq // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_query_count(self.h, _p(q), nq, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), nq, _p(ptr), _p(scratch), None) == 0
        idx = np.zeros(max(int(ptr[-1]), 1), dtype=np.int32)
        assert lib.dsk_lsh_query_fill(self.h, _p(q), nq, _p(ptr), _p(idx), None) == 0, lib.dsk_last_error()
        return ptr, idx[:int(ptr[-1])]

    def close(self):
        self.lib.dsk_lsh_destroy(self.h)


class _Emu:
    grid_rows = 2          # the emulated device has two SMs
    name = "emu"

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuIndex(self.lib, k, b, r, capacity)

    def fingerprints(self, sig, b, r):
        sig = _aligned(np.asarray(sig, dtype=np.uint32))
        fp = np.zeros((len(sig), b), dtype=np.uint64)
        assert self.lib.dsk_band_fingerprints(_p(sig), len(sig), sig.shape[1], b, r, _p(fp), None) == 0
        return fp

    def workspace_size(self, nq, n, k):
        return int(self.lib.dsk_jaccard_topk_workspace_size(nq, n, k))

    def topk(self, q, db, topk, self_base, prefilter):
        lib = self.lib
        q, db = _aligned(np.asarray(q, dtype=np.uint32)), _aligned(np.asarray(db, dtype=np.uint32))
        (nq, k), n = q.shape, len(db)
        cnt, idx = np.zeros((nq, topk), dtype=np.int32), np.zeros((nq, topk), dtype=np.int64)
        ws_bytes = self.workspace_size(nq, n, k) if prefilter else 0
        ws = _aligned(np.zeros(max(ws_bytes, 16), dtype=np.uint8))
        rc = lib.dsk_jaccard_topk_ws(_p(q), nq, _p(db), n, k, topk, self_base, _p(cnt), _p(idx),
                                     _p(ws) if ws_bytes else None, ws_bytes, None)
        if rc != 0:
            raise RuntimeError(lib.dsk_last_error().decode())
        return cnt, idx


class _GpuIndex:
    def __init__(self, dsk, k, b, r, capacity):
        self.ix = dsk.GpuLSH(num_perm=k, params=(b, r), capacity=capacity)

    def insert(self, sig):
        self.ix.insert(np.ascontiguousarray(sig, dtype=np.uint32))

    def insert_tokens(self, tok, off, perms):
        import torch
        self.ix.insert_tokens(torch.from_numpy(np.ascontiguousarray(tok).view(np.int32)).cuda(),
                              torch.from_numpy(np.ascontiguousarray(off)).cuda(), len(tok), perms)

    def query(self, q):
        return self.ix.query(np.ascontiguousarray(q, dtype=np.uint32))

    def close(self):
        pass


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk
        self.grid_rows = dsk._native.device_info(0)["sm_count"]

    def index(self, k, b, r, capacity):
        return _GpuIndex(self.dsk, k, b, r, capacity)

    def fingerprints(self, sig, b, r):
        return self.dsk.codec.band_fingerprints(np.ascontiguousarray(sig, dtype=np.uint32), b, r).cpu().numpy().view(np.uint64)

    def workspace_size(self, nq, n, k):
        return int(self.dsk._native.load().dsk_jaccard_topk_workspace_size(nq, n, k))

    def topk(self, q, db, topk, self_base, prefilter):
        c, i = self.dsk.codec.jaccard_topk(np.ascontiguousarray(q, dtype=np.uint32), np.ascontiguousarray(db, dtype=np.uint32),
                                           topk=topk, self_base=self_base, to_host=False, prefilter=prefilter)
        return c.cpu().numpy(), i.cpu().numpy()


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- helpers -----------------------------------------------------------------------------------------------------------
def _rand(rng, *shape):
    return rng.randint(0, 1 << 32, size=shape, dtype=np.uint64).astype(np.uint32)


def _assert_candidates_equal_oracle(ix, rows, k, b, r, queries):
    """``rows`` in insertion order (document i = row i); every query's candidates as a set == DictLSH's."""
    ref = o.DictLSH(k, b, r)
    for i, row in enumerate(rows):
        ref.insert(i, row.astype(np.uint64))
    ptr, idx = ix.query(queries)
    for j, q in enumerate(queries):
        got = idx[ptr[j]:ptr[j + 1]].tolist()
        assert len(got) == len(set(got)), j                            # each candidate once (union over bands)
        assert sorted(got) == sorted(ref.query(q.astype(np.uint64))), j


def _assert_collide(be, pairs, b, r):
    """Each (row_a, row_b, band): different tuples in that band, same fingerprint in the library and in the model."""
    assert pairs
    a = np.stack([p[0] for p in pairs])
    c = np.stack([p[1] for p in pairs])
    bands = np.array([p[2] for p in pairs])
    fa, fc = be.fingerprints(a, b, r), be.fingerprints(c, b, r)
    assert np.array_equal(fa, hm.band_fp(a, b, r)) and np.array_equal(fc, hm.band_fp(c, b, r))
    sel = np.arange(len(pairs))
    assert np.array_equal(fa[sel, bands], fc[sel, bands])
    for (x, y, j) in pairs:
        assert not np.array_equal(x[j * r:(j + 1) * r], y[j * r:(j + 1) * r])


def _colliders(rng, sig, band, r, want):
    """Up to ``want`` (doc, tuple) pairs: a tuple different from sig[doc]'s band tuple with the same fingerprint."""
    out = []
    for d in rng.permutation(len(sig)):
        t = hm.second_preimage(sig[d, band * r:(band + 1) * r], band, rng)
        if t is not None:
            out.append((int(d), t))
            if len(out) == want:
                break
    return out


# ---- the model is the library's hash ------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,b,r", [(128, 9, 13), (128, 40, 3), (64, 32, 2), (16, 16, 1), (256, 17, 15)])
def test_band_fingerprint_model_equals_the_library(be, k, b, r):
    """dsk_band_fingerprints (band_fingerprint_kernel) == hash_model.band_fp bit for bit, including the remap of a
    tuple whose fingerprint is the tables' empty key (r >= 2; for r = 1 no value reaches it)."""
    rng = np.random.RandomState(k + b + r)
    sig = _rand(rng, 301, k)
    if r >= 2:
        for j in range(b):
            e = hm.tuple_with_prefp(hm.EMPTY_KEY, j, r, rng)
            if e is not None:
                sig[5, j * r:(j + 1) * r] = e
                assert hm.lsh_mix64(hm.tuple_states(e[None], j))[0] == hm.EMPTY_KEY
                break
        else:
            pytest.fail("no empty-key tuple found")
    want = hm.band_fp(sig, b, r)
    assert np.array_equal(be.fingerprints(sig, b, r), want)
    if r >= 2:
        assert (want == np.uint64(hm.EMPTY_KEY - 1)).sum() == 1 and not (want == np.uint64(hm.EMPTY_KEY)).any()


# ---- LSH: colliding tuples --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,b,r", [(128, 40, 3), (64, 32, 2), (128, 9, 13)])
def test_lsh_colliding_tuples_are_told_apart(be, k, b, r):
    """Documents whose band tuple collides with another document's, as inserted documents and as queries, several
    colliders in one chain, bands in both lane rounds of the query kernel (b = 40); documents that collide with the
    query in one band and truly match it in a later band (the cross-band de-duplication must compare tuples)."""
    rng = np.random.RandomState(k * b + r)
    base = _rand(rng, 160, k)
    bands = sorted({0, 1, b // 2, b - 1} | ({32, 35} if b > 32 else set()))
    extra, queries, pairs = [], [], []
    for band in bands:
        sl = slice(band * r, (band + 1) * r)
        for d, t in _colliders(rng, base, band, r, 3):
            x = _rand(rng, k)                        # collides with document d in this band, nothing else
            x[sl] = t
            extra.append(x)
            pairs.append((base[d], x, band))
            t2 = hm.second_preimage(base[d, sl], band, rng, avoid=[t])
            if t2 is not None:                       # a third member of the same chain
                y = _rand(rng, k)
                y[sl] = t2
                extra.append(y)
                pairs.append((base[d], y, band))
            q = _rand(rng, k)                        # query: equal to x's tuple, colliding with d's
            q[sl] = t
            queries.append(q)
            later = [j for j in range(band + 1, b)]
            if later:                                # collides with d in `band`, truly matches d in a later band
                j2 = int(rng.choice(later))
                z = _rand(rng, k)
                z[sl] = t
                z[j2 * r:(j2 + 1) * r] = base[d, j2 * r:(j2 + 1) * r]
                extra.append(z)
                pairs.append((base[d], z, band))
                w = _rand(rng, k)                    # the same seen from the query side
                w[sl] = t
                w[j2 * r:(j2 + 1) * r] = base[d, j2 * r:(j2 + 1) * r]
                queries.append(w)
    assert len(pairs) >= 2 * len(bands)
    _assert_collide(be, pairs, b, r)
    extra = np.stack(extra)
    h = len(extra) // 2
    rows = np.concatenate([extra[:h], base, extra[h:]])
    ix = be.index(k, b, r, len(rows))
    for part in (extra[:h], base[:80], base[80:], extra[h:]):
        ix.insert(part)
    try:
        _assert_candidates_equal_oracle(ix, rows, k, b, r, np.concatenate([base, extra, np.stack(queries)]))
    finally:
        ix.close()


@pytest.mark.parametrize("r", [2, 3])
def test_lsh_empty_key_tuple_keeps_its_bucket(be, r):
    """A tuple whose fingerprint is the tables' empty key (remapped to EMPTY_KEY - 1) next to a tuple whose fingerprint
    is EMPTY_KEY - 1: one bucket, told apart by the tuples.  Tuples whose home slot is the empty key's home slot (and
    the remapped key's) are inserted after it: without the remap the empty-key insert would leave its slot looking
    empty, a later tuple would claim it and the empty-key documents would be lost."""
    b, k, capacity = 16, 16 * r, 300
    rng = np.random.RandomState(40 + r)
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, r, rng)
        z = hm.tuple_with_prefp(hm.EMPTY_KEY - 1, band, r, rng)
        if e is not None and z is not None:
            break
    else:
        pytest.fail("no band with both tuples")
    sl = slice(band * r, (band + 1) * r)
    cand = _rand(rng, 1 << 17, r)
    home = hm.home_slot(hm.tuple_fp(cand, band), capacity)
    same = [cand[home == hm.home_slot(np.uint64(key), capacity)][:4] for key in (hm.EMPTY_KEY, hm.EMPTY_KEY - 1)]
    assert all(len(s) == 4 for s in same)

    def with_tuple(t):
        x = _rand(rng, k)
        x[sl] = t
        return x

    e_rows = np.stack([with_tuple(e) for _ in range(3)])
    z_rows = np.stack([with_tuple(z) for _ in range(2)])
    y_rows = np.stack([with_tuple(t) for t in np.concatenate(same)])
    base = _rand(rng, 60, k)
    fp = be.fingerprints(np.stack([e_rows[0], z_rows[0]]), b, r)[:, band]
    assert (fp == np.uint64(hm.EMPTY_KEY - 1)).all()
    assert hm.lsh_mix64(hm.tuple_states(e[None], band))[0] == hm.EMPTY_KEY
    groups = [base[:30], e_rows[:1], z_rows[:1], y_rows, e_rows[1:], z_rows[1:], base[30:]]
    rows = np.concatenate(groups)
    ix = be.index(k, b, r, capacity)
    for g in groups:
        ix.insert(g)
    try:
        extra_q = np.stack([with_tuple(e), with_tuple(z), with_tuple(same[0][0])])
        _assert_candidates_equal_oracle(ix, rows, k, b, r, np.concatenate([rows, extra_q]))
    finally:
        ix.close()


def test_lsh_probe_cluster_wraps_past_the_table_end(be):
    """r = 1: many distinct values of one band whose home slots are the table's last 8 slots, so their probes wrap to
    slot 0; queries for the cluster's members and for absent values whose probe sequence crosses the cluster."""
    k = b = 16
    r, capacity, band = 1, 400, 3
    mask = hm.cap_slots(capacity) - 1
    rng = np.random.RandomState(11)
    vals = np.unique(_rand(rng, 1 << 20))
    home = hm.home_slot(hm.tuple_fp(vals[:, None], band), capacity)
    tail = vals[home >= mask - 7]
    members, absent = tail[:48], tail[48:88]
    near0 = vals[home < 16][:20]                  # home slots the wrapped cluster covers
    assert len(members) == 48 and len(absent) == 40 and len(near0) == 20

    def rows_with(vs):
        x = _rand(rng, len(vs), k)
        x[:, band] = vs
        return x

    docs = rows_with(np.concatenate([members, members[:3]]))      # three buckets of two members
    rng.shuffle(docs)
    ix = be.index(k, b, r, capacity)
    ix.insert(docs[:25])
    ix.insert(docs[25:])
    try:
        q = np.concatenate([docs, rows_with(members), rows_with(absent), rows_with(near0)])
        _assert_candidates_equal_oracle(ix, docs, k, b, r, q)
    finally:
        ix.close()


def test_lsh_fused_token_insert_shares_chains_with_plain_insert(be):
    """Documents inserted from tokens (dsk_lsh_insert_tokens' fused route: K = 128 <= 256, u32 tokens, seeded
    permutations) and rows inserted with plain insert before and after them whose band tuples collide with the token
    documents' (the signatures are known in advance from the C oracle): chains that mix rows from the signature kernel's
    insert epilogue and from lsh_insert_kernel, bands >= 32 included."""
    k, b, r = 128, 40, 3
    rng = np.random.RandomState(8)
    n = 90
    lens = rng.randint(1, 150, size=n)
    lens[::9] = 0
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = _rand(rng, int(off[-1]))
    for d in range(4, n, 11):                     # exact duplicates: buckets with several token documents
        a0, a1 = int(off[d - 1]), int(off[d])
        if a1 - a0 == lens[d] and lens[d] > 0:
            tok[off[d]:off[d + 1]] = tok[a0:a1]
    perms = o.init_permutations(k, 5)
    sig = oc.minhash_bulk_u32tok(tok, off, perms)
    colliders, pairs, queries = [], [], []
    for band in (0, 7, 31, 32, 39):
        sl = slice(band * r, (band + 1) * r)
        for d, t in _colliders(rng, sig[lens > 0], band, r, 3):
            d = int(np.nonzero(lens > 0)[0][d])
            x = _rand(rng, k)
            x[sl] = t
            if band < 32:                         # and truly matches the token document in a later band
                j2 = band + 5
                x[j2 * r:(j2 + 1) * r] = sig[d, j2 * r:(j2 + 1) * r]
            colliders.append(x)
            pairs.append((sig[d], x, band))
            q = _rand(rng, k)
            q[sl] = t
            queries.append(q)
    _assert_collide(be, pairs, b, r)
    colliders = np.stack(colliders)
    h = len(colliders) // 2
    ix = be.index(k, b, r, n + len(colliders))
    ix.insert(colliders[:h])
    ix.insert_tokens(tok, off, perms)
    ix.insert(colliders[h:])
    rows = np.concatenate([colliders[:h], sig, colliders[h:]])
    try:
        _assert_candidates_equal_oracle(ix, rows, k, b, r, np.concatenate([sig, colliders, np.stack(queries)]))
    finally:
        ix.close()


# ---- top-k: fingerprint twins, shared-memory limits, grid-stride loops ---------------------------------------------------
def _brute_topk(q, db, topk, self_base):
    cnt_out = np.full((len(q), topk), -1, dtype=np.int64)
    idx_out = np.full((len(q), topk), -1, dtype=np.int64)
    for i, row in enumerate(q):
        cnt = (db == row[None, :]).sum(axis=1)
        order = np.lexsort((np.arange(len(db)), -cnt))               # count desc, index asc
        if self_base >= 0:
            order = order[order != self_base + i]
        order = order[:topk]
        cnt_out[i, :len(order)] = cnt[order]
        idx_out[i, :len(order)] = order
    return cnt_out, idx_out


def _twin_db(rng, q, n):
    """Database rows that are fingerprint twins of a query in every position (bound = K) but equal to it in at most 3;
    the true near-duplicates (K - 1 .. K - 6 equal, in tied pairs) at the highest indices."""
    nq, k = q.shape
    owner = np.arange(n) % nq
    db = hm.fp16_twins(q[owner], rng)
    for i in range(0, n, 3):
        pos = rng.choice(k, int(rng.randint(1, 4)), replace=False)
        db[i, pos] = q[owner[i], pos]
    for t in range(24):
        i = n - 24 + t
        owner[i] = (t // 2) * 5 % nq
        db[i] = q[owner[i]]
        pos = rng.choice(k, 1 + t // 4, replace=False)
        db[i, pos] = hm.fp16_twins(db[i, pos], rng)
        if t % 2:
            db[i] = db[i - 1]                    # exact tie with the row before it
    return db, owner


@pytest.mark.parametrize("k", [32, 100, 480, 481, 512, 513, 736, 737, 1024, 4096])
def test_topk_fingerprint_twins_and_every_num_perm(be, k):
    """Most database rows agree with a query in all K fingerprints but in few values: the prefilter must count them
    exactly.  K from 32 to 4096 (the C-ABI's limit) on both sides of the shared-memory limits of the prefilter tile
    (K = 480) and of the exact kernel's resident query tile (K = 736); n >= 512 so the prefilter engages where it fits;
    n and nq not multiples of the tiles.  prefilter on and off, topk = 1, 7, 32."""
    rng = np.random.RandomState(k)
    n, nq = 600, 70
    q = _rand(rng, nq, k)
    db, owner = _twin_db(rng, q, n)
    bound = (hm.topk_fp16(db) == hm.topk_fp16(q[owner])).sum(axis=1)
    exact = (db == q[owner]).sum(axis=1)
    assert (bound == k).sum() > 0.9 * n and (exact <= 3).sum() > 0.9 * n
    assert (be.workspace_size(nq, n, k) > 0) == (k <= 480)
    for topk in ((1, 7, 32) if be.name == "gpu" else (1, 32)):     # the emulated prefilter is slow
        want_c, want_i = _brute_topk(q, db, topk, -1)
        for prefilter in (True, False):
            c, i = be.topk(q, db, topk, -1, prefilter)
            assert np.array_equal(i, want_i), (topk, prefilter)
            assert np.array_equal(c, want_c), (topk, prefilter)


@pytest.mark.parametrize("k", [128, 100])
def test_topk_grid_stride_over_query_tiles(be, k):
    """More query tiles than the grid has CTAs (2 x SMs tiles of 64 queries with the prefilter, 3 x SMs without), so
    both kernels' grid-stride loops run more than once; queries are database rows (self_base > 0) with twins and
    near-duplicates planted next to them.  A sample of queries and every query of the last tile are checked."""
    rng = np.random.RandomState(k + 1)
    nq = 7 * 64 * be.grid_rows // 2 + 5 if be.name == "emu" else 40_037
    base = 3
    n = nq + base + 300
    db = _rand(rng, n, k)
    db[1::2] = hm.fp16_twins(db[0::2][: n // 2], rng)
    near = rng.randint(0, n, size=n // 10)
    db[near, : k // 2] = db[(near + 7) % n, : k // 2]
    q = db[base:base + nq]
    assert -(-nq // 64) > 3 * be.grid_rows
    last = (nq - 1) // 64 * 64
    check = np.unique(np.concatenate([rng.choice(last, 150, replace=False), np.arange(last, nq)]))
    want_c = np.full((len(check), 10), -1, dtype=np.int64)
    want_i = np.full((len(check), 10), -1, dtype=np.int64)
    for j, qi in enumerate(check):
        c1, i1 = _brute_topk(q[qi:qi + 1], db, 10, base + qi)
        want_c[j], want_i[j] = c1[0], i1[0]
    assert be.workspace_size(nq, n, k) > 0
    for prefilter in (True, False):
        c, i = be.topk(q, db, 10, base, prefilter)
        assert np.array_equal(i[check], want_i), prefilter
        assert np.array_equal(c[check], want_c), prefilter
