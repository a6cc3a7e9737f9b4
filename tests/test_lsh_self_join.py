"""GpuLSH.candidate_pairs / duplicate_clusters: the self-join of a device-resident LSH index.

Documents i and d < i are a candidate pair iff d is in MinHashLSH.query(row i) (an equal r-tuple in some band,
lsh.py:370-432); ``eq`` counts the positions where the rows agree, so eq / K is MinHash.jaccard (minhash.py:324), and
``min_jaccard`` keeps the pairs with MinHash.jaccard >= min_jaccard.  Clusters are the connected components of the
kept pairs, labelled by their smallest document.

The oracle is composed here from the dict-bucket index (oracle_np.DictLSH.query), oracle_np.jaccard and scipy's
connected_components.  Every case runs on two backends: ``emu``, the whole library compiled with g++ on the emulation
shim (tests/emu/emu_capi.cpp, two emulated SMs) and driven through its C-ABI, and ``gpu``, the compiled library on the
H100 through the Python API.
"""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from oracle import oracle_clib as oc
from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
DSK_OK, DSK_ERR_INVALID = 0, 1


def _min_count(min_jaccard, k):
    from datasketch_b200.lsh import _jaccard_min_count
    return _jaccard_min_count(min_jaccard, k)


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
        self.lib, self.k, self.n = lib, k, 0
        self.h = ctypes.c_void_p()
        assert lib.dsk_lsh_create(k, b, r, capacity, 0, ctypes.byref(self.h)) == 0, lib.dsk_last_error()

    def insert(self, sig):
        sig = _aligned(np.asarray(sig, dtype=np.uint32))
        assert self.lib.dsk_lsh_insert(self.h, _p(sig), len(sig), None) == 0, self.lib.dsk_last_error()
        self.n += len(sig)

    def insert_tokens(self, tok, off, perms):
        lib, ph = self.lib, ctypes.c_void_p()
        a, b = np.ascontiguousarray(perms[0]), np.ascontiguousarray(perms[1])
        assert lib.dsk_perm_create(_p(a), _p(b), self.k, 0, ctypes.byref(ph)) == 0, lib.dsk_last_error()
        tok, off = _aligned(tok), _aligned(off)
        rc = lib.dsk_lsh_insert_tokens(self.h, ph, _p(tok), 0, _p(off), len(off) - 1, len(tok), None)
        lib.dsk_perm_destroy(ph)
        assert rc == 0, lib.dsk_last_error()
        self.n += len(off) - 1

    def pairs(self, min_jaccard=None):
        lib, n, mc = self.lib, self.n, _min_count(min_jaccard, self.k)
        counts, ptr = np.zeros(n + 1, dtype=np.int64), np.zeros(n + 1, dtype=np.int64)
        scratch = np.zeros(n // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_pairs_count(self.h, mc, _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), n, _p(ptr), _p(scratch), None) == 0
        m = int(ptr[-1])
        idx, eq = np.full(max(m, 1), -1, dtype=np.int32), np.full(max(m, 1), -1, dtype=np.int32)
        assert lib.dsk_lsh_pairs_fill(self.h, mc, _p(ptr), _p(idx), _p(eq), None) == 0, lib.dsk_last_error()
        return ptr, idx[:m], eq[:m]

    def clusters(self, min_jaccard=None):
        labels = np.full(max(self.n, 1), -7, dtype=np.int32)
        rc = self.lib.dsk_lsh_clusters(self.h, _min_count(min_jaccard, self.k), _p(labels), None)
        assert rc == 0, self.lib.dsk_last_error()
        return labels[:self.n]

    def close(self):
        self.lib.dsk_lsh_destroy(self.h)


class _Emu:
    name = "emu"
    grid_docs = 2 * 8 * 8          # two emulated SMs x 8 CTAs x 8 warps: documents one sweep of the pair walk covers

    def __init__(self, lib):
        self.lib = lib

    def index(self, k, b, r, capacity):
        return _EmuIndex(self.lib, k, b, r, capacity)


class _GpuIndex:
    def __init__(self, dsk, k, b, r, capacity):
        self.ix = dsk.GpuLSH(num_perm=k, params=(b, r), capacity=capacity)

    def insert(self, sig):
        self.ix.insert(np.ascontiguousarray(sig, dtype=np.uint32))

    def insert_tokens(self, tok, off, perms):
        import torch
        self.ix.insert_tokens(torch.from_numpy(np.ascontiguousarray(tok).view(np.int32)).cuda(),
                              torch.from_numpy(np.ascontiguousarray(off)).cuda(), len(tok), perms)

    def pairs(self, min_jaccard=None):
        return self.ix.candidate_pairs(min_jaccard)

    def clusters(self, min_jaccard=None):
        return self.ix.duplicate_clusters(min_jaccard)

    def close(self):
        pass


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.dsk = dsk
        self.grid_docs = dsk._native.device_info(0)["sm_count"] * 8 * 8

    def index(self, k, b, r, capacity):
        return _GpuIndex(self.dsk, k, b, r, capacity)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- oracle ------------------------------------------------------------------------------------------------------------
def _oracle_pairs(rows, k, b, r, min_jaccard):
    """{(i, d): eq} for d < i in DictLSH.query(row i) with oracle_np.jaccard >= min_jaccard (None: all)."""
    rows = np.asarray(rows, dtype=np.uint64)
    ref = o.DictLSH(k, b, r)
    for i, row in enumerate(rows):
        ref.insert(i, row)
    out = {}
    for i, row in enumerate(rows):
        for d in ref.query(row):
            if d < i and (min_jaccard is None or o.jaccard(row, rows[d]) >= min_jaccard):
                out[(i, d)] = int(np.count_nonzero(row == rows[d]))
    return out


def _components(n, pairs):
    """labels[i] = smallest document of i's connected component (scipy connected_components of the pair graph)."""
    e = np.array(list(pairs), dtype=np.int64).reshape(-1, 2)
    g = coo_matrix((np.ones(len(e), dtype=np.int8), (e[:, 0], e[:, 1])), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    first = np.full(comp.max() + 1 if n else 0, n, dtype=np.int64)
    np.minimum.at(first, comp, np.arange(n))
    return first[comp]


def _pairs_dict(ptr, idx, eq):
    n = len(ptr) - 1
    assert ptr[0] == 0 and np.all(np.diff(ptr) >= 0) and ptr[-1] == len(idx) == len(eq)
    rows = np.repeat(np.arange(n), np.diff(ptr))
    got = dict(zip(zip(rows.tolist(), idx.tolist()), eq.tolist()))
    assert len(got) == len(idx)                                   # each unordered pair once
    return got


def _check(ix, rows, k, b, r, thresholds=(None, 0.0, 0.5, 1.0)):
    n = len(rows)
    for t in thresholds:
        want = _oracle_pairs(rows, k, b, r, t)
        got = _pairs_dict(*ix.pairs(t))
        assert got == want, t
        labels = ix.clusters(t)
        assert labels.dtype == np.int32 and len(labels) == n
        assert np.array_equal(labels, _components(n, want)), t


def _low_entropy(rs, n, k, vals):
    sig = rs.randint(0, vals, size=(n, k)).astype(np.uint32)
    sig[rs.randint(0, n, n // 8)] = sig[rs.randint(0, n, n // 8)]         # exact duplicates
    return sig


# ---- cases -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,b,r,vals,t", [(32, 8, 4, 3, 0.37), (128, 40, 3, 4, 0.3), (100, 33, 3, 4, 0.29)])
def test_low_entropy_big_buckets_two_batches(be, k, b, r, vals, t):
    """Few distinct values: big buckets, pairs that match in several bands (emitted once, by the first), exact
    duplicate rows, b > 32 bands (two lane rounds), two insert batches, more documents than one sweep of the grid.
    min_jaccard: none, 0.0, a value that is not a multiple of 1/K, 0.5 and 1.0 (the exact duplicates)."""
    rs = np.random.RandomState(k + b)
    n = 3 * be.grid_docs + 11 if be.name == "emu" else 2500
    if be.name == "emu" and b > 32:
        n = be.grid_docs + 37               # the emulated pair walk over these buckets is slow
    sig = _low_entropy(rs, n, k, vals)
    assert t * k != int(t * k)
    ix = be.index(k, b, r, n + 3)
    ix.insert(sig[:n // 3])
    ix.insert(sig[n // 3:])
    try:
        _check(ix, sig, k, b, r, (None, 0.0, t, 0.5, 1.0))
    finally:
        ix.close()


def test_planted_near_duplicates_grid_stride(be):
    """Random rows with planted near-duplicates (a copy with a few positions redrawn, chains of copies), many more
    documents than the grid covers in one sweep, so the pair walk's and the link kernel's grid-stride loops run."""
    k, b, r = 128, 16, 8
    rs = np.random.RandomState(17)
    n = 5 * be.grid_docs + 3 if be.name == "emu" else 40_000
    sig = rs.randint(0, 1 << 32, size=(n, k), dtype=np.uint64).astype(np.uint32)
    dst = rs.choice(n, n // 5, replace=False)
    for d in dst:
        s = int(rs.randint(0, n))
        sig[d] = sig[s]
        pos = rs.choice(k, int(rs.randint(0, 40)), replace=False)
        sig[d, pos] = rs.randint(0, 1 << 32, size=len(pos), dtype=np.uint64).astype(np.uint32)
    ix = be.index(k, b, r, n)
    ix.insert(sig)
    try:
        _check(ix, sig, k, b, r, (None, 0.8, 0.9))
    finally:
        ix.close()


def test_rows_from_the_fused_token_insert(be):
    """Documents inserted from tokens (dsk_lsh_insert_tokens' fused route: the signature kernel's insert epilogue)
    between two plain inserts of near-duplicate rows of them: the self-join reads the rows the epilogue wrote."""
    k, b, r = 128, 32, 4
    rs = np.random.RandomState(5)
    n = 120 if be.name == "emu" else 3000
    lens = rs.randint(1, 200, size=n)
    lens[::13] = 0
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, 1 << 32, size=int(off[-1]), dtype=np.uint64).astype(np.uint32)
    for d in range(5, n, 7):                                    # near-duplicate documents: a copy with a few tokens redrawn
        s = int(rs.randint(0, d))
        if lens[d] == lens[s] and lens[d] > 0:
            tok[off[d]:off[d + 1]] = tok[off[s]:off[s + 1]]
            tok[off[d] + rs.randint(0, lens[d], size=1 + lens[d] // 30)] = rs.randint(0, 1 << 32, dtype=np.uint64)
        elif lens[d] == lens[d - 1]:
            tok[off[d]:off[d + 1]] = tok[off[d - 1]:off[d]]
    perms = o.init_permutations(k, 5)
    sig = oc.minhash_bulk_u32tok(tok, off, perms)
    before = sig[rs.choice(n, 20, replace=False)].copy()
    after = sig[rs.choice(n, 20, replace=False)].copy()
    after[:, : k // 4] = rs.randint(0, 1 << 32, size=(20, k // 4), dtype=np.uint64).astype(np.uint32)
    ix = be.index(k, b, r, n + 40)
    ix.insert(before)
    ix.insert_tokens(tok, off, perms)
    ix.insert(after)
    rows = np.concatenate([before, sig, after])
    try:
        assert sum(1 for _ in _oracle_pairs(rows, k, b, r, 0.9)) >= 10      # the planted duplicates meet
        _check(ix, rows, k, b, r, (None, 0.7, 0.9))
    finally:
        ix.close()


def test_one_document_and_empty_index(be):
    k, b, r = 64, 8, 8
    ix = be.index(k, b, r, 10)
    try:
        ptr, idx, eq = ix.pairs()
        assert list(ptr) == [0] and len(idx) == 0 and len(eq) == 0
        assert len(ix.clusters()) == 0 and len(ix.clusters(0.5)) == 0
        ix.insert(np.arange(k, dtype=np.uint32)[None])
        for t in (None, 0.0, 1.0):
            ptr, idx, eq = ix.pairs(t)
            assert list(ptr) == [0, 0] and len(idx) == 0
            assert ix.clusters(t).tolist() == [0]
    finally:
        ix.close()


@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_in_a_chain(be, head_collides):
    """Members of one bucket chain whose tuples differ but share the band's fingerprint (second preimages from
    tests/hash_model.py), and tuples whose fingerprint is the tables' empty key: the pair walk must not pair them and
    the link kernel must skip them -- also when the chain's head (its most recently inserted member) is such a member."""
    k, b, r = 96, 32, 3
    rs = np.random.RandomState(23 + head_collides)
    n_base = 150
    base = rs.randint(0, 1 << 32, size=(n_base, k), dtype=np.uint64).astype(np.uint32)
    groups, colliders = [], []
    for band in (0, 5, 31):
        sl = slice(band * r, (band + 1) * r)
        for d in rs.permutation(n_base)[:40]:
            t2 = hm.second_preimage(base[d, sl], band, rs)
            if t2 is None:
                continue
            same = base[rs.randint(0, n_base, 2)].copy()           # two more members with d's tuple
            same[:, sl] = base[d, sl]
            other = base[rs.randint(0, n_base, 2)].copy()          # two with the colliding tuple: a pair of their own
            other[:, sl] = t2
            groups.append(same)
            colliders.append(other)
            break
        else:
            pytest.fail("no second preimage found for band %d" % band)
    e = None
    for band in range(b):
        e = hm.tuple_with_prefp(hm.EMPTY_KEY, band, r, rs)
        if e is not None:
            empty = base[rs.randint(0, n_base, 3)].copy()
            empty[:, band * r:(band + 1) * r] = e
            groups.append(empty)
            break
    assert e is not None
    fp = hm.band_fp(np.concatenate(colliders + groups), b, r)
    assert len(np.unique(fp)) < fp.size                               # the colliders really share fingerprints
    extra = np.concatenate(groups)
    coll = np.concatenate(colliders)
    parts = [base, extra, coll] if head_collides else [base, coll, extra]
    rows = np.concatenate(parts)
    ix = be.index(k, b, r, len(rows))
    for p in parts:
        ix.insert(p)
    try:
        want = _oracle_pairs(rows, k, b, r, None)
        n0, n1 = n_base, n_base + len(parts[1])
        assert any(i >= n1 and d < n1 for (i, d) in want) or any(i >= n0 and d < n0 for (i, d) in want)
        _check(ix, rows, k, b, r, (None, 0.0, 0.05))
    finally:
        ix.close()


def test_c_abi_argument_validation(emu_lib):
    """Null handle, min_count outside [0, K], null buffers of a non-empty index: DSK_ERR_INVALID, nothing launched."""
    lib, k = emu_lib, 32
    buf = np.zeros(64, dtype=np.int64)
    for fn, args in ((lib.dsk_lsh_pairs_count, (_p(buf),)), (lib.dsk_lsh_pairs_fill, (_p(buf), _p(buf), _p(buf))),
                     (lib.dsk_lsh_clusters, (_p(buf),))):
        assert fn(None, 0, *args, None) == DSK_ERR_INVALID
        assert b"null handle" in lib.dsk_last_error()
    ix = _EmuIndex(lib, k, 8, 4, 20)
    try:
        nulls = [(lib.dsk_lsh_pairs_count, (None,)), (lib.dsk_lsh_pairs_fill, (None, None, None)),
                 (lib.dsk_lsh_clusters, (None,))]
        for fn, args in nulls:                              # empty index: nothing to write, null buffers are fine
            assert fn(ix.h, 0, *args, None) == DSK_OK
        ix.insert(np.arange(3 * k, dtype=np.uint32).reshape(3, k) % 5)
        for fn, args in nulls:
            assert fn(ix.h, 0, *args, None) == DSK_ERR_INVALID
            assert b"null buffer" in lib.dsk_last_error()
        for j in range(3):                                  # one null buffer of the fill is enough to refuse it
            args = [_p(buf)] * 3
            args[j] = None
            assert lib.dsk_lsh_pairs_fill(ix.h, 0, *args, None) == DSK_ERR_INVALID
        good = [(lib.dsk_lsh_pairs_count, (_p(buf),)), (lib.dsk_lsh_pairs_fill, (_p(buf), _p(buf), _p(buf))),
                (lib.dsk_lsh_clusters, (_p(buf),))]
        for fn, args in good:
            for mc in (-1, k + 1, -(1 << 31)):
                assert fn(ix.h, mc, *args, None) == DSK_ERR_INVALID
                assert b"min_count" in lib.dsk_last_error()
        for mc in (0, k):
            assert lib.dsk_lsh_clusters(ix.h, mc, _p(buf), None) == DSK_OK
    finally:
        ix.close()


@pytest.mark.parametrize("k", [16, 100, 128, 256])
def test_min_jaccard_to_min_count_is_the_reference_division(k):
    """min_count = the smallest c with float(c) / float(K) >= min_jaccard, for every c (and the neighbouring floats)."""
    for c in range(k + 1):
        t = float(c) / float(k)
        assert _min_count(t, k) == c
        if c < k:
            assert _min_count(float(np.nextafter(t, 2.0)), k) == c + 1
        if c > 0:
            assert _min_count(float(np.nextafter(t, -1.0)), k) == c
    rs = np.random.RandomState(k)
    counts = np.arange(k + 1)
    for t in rs.rand(200):
        assert _min_count(float(t), k) == int(counts[counts / float(k) >= t][0])
    assert _min_count(None, k) == 0 and _min_count(0.0, k) == 0 and _min_count(1.0, k) == k
    for bad in (-0.01, 1.0000001, float("nan"), 2.0):
        with pytest.raises(ValueError):
            _min_count(bad, k)


def test_thread_sanitizer_union_find():
    """Both cluster paths under ThreadSanitizer (tests/emu/emu_tsan_clusters_main.cpp, linked with the whole emulated
    library): hundreds of host threads hook roots of one big component at once; every load and store of a parent that
    races with a hook must be atomic, or TSan reports a data race.  The labels are also checked against a serial
    union-find of brute-force pairs."""
    out = os.path.join(EMU, "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "emu_tsan_clusters")
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-ffp-contract=off", "-fsanitize=thread", "-DDSK_EMU",
                            "-I" + EMU, "-o", exe, os.path.join(EMU, "emu_capi.cpp"),
                            os.path.join(EMU, "emu_tsan_clusters_main.cpp")], capture_output=True, text=True)
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
def test_pairs_equal_the_reference_query_golden(golden):
    """tests/golden/lsh.npz: 300 signatures and the candidate lists the reference's MinHashLSH.query returned for each
    (threshold 0.8, K = 128).  candidate_pairs() must be exactly {(i, d): d in query(i), d < i}, eq the oracle's count."""
    import datasketch_b200 as dsk
    g = golden("lsh")
    sig, qp, qi = g["sig"], g["query_ptr"], g["query_idx"]
    ix = dsk.GpuLSH(threshold=0.8, num_perm=128, capacity=len(sig))
    assert [ix.b, ix.r] == g["b_r"].tolist()
    ix.insert(sig)
    want = {}
    for i in range(len(sig)):
        for d in qi[qp[i]:qp[i + 1]].tolist():
            if d < i:
                want[(i, d)] = int(np.count_nonzero(sig[i] == sig[d]))
    assert want
    assert _pairs_dict(*ix.candidate_pairs()) == want
    assert np.array_equal(ix.duplicate_clusters(), _components(len(sig), want))
    for t in (0.3, 0.8):
        w = {p: e for p, e in want.items() if o.jaccard(sig[p[0]].astype(np.uint64), sig[p[1]].astype(np.uint64)) >= t}
        assert _pairs_dict(*ix.candidate_pairs(t)) == w
        assert np.array_equal(ix.duplicate_clusters(t), _components(len(sig), w))
    import torch
    ptr, idx, eq = ix.candidate_pairs(to_host=False)
    assert ptr.is_cuda and ptr.dtype == torch.int64 and idx.dtype == torch.int32 and eq.dtype == torch.int32
    labels = ix.duplicate_clusters(to_host=False)
    assert labels.is_cuda and labels.dtype == torch.int32
    for bad in (-0.5, 1.5):
        with pytest.raises(ValueError):
            ix.candidate_pairs(bad)
        with pytest.raises(ValueError):
            ix.duplicate_clusters(bad)


@pytest.mark.gpu
def test_c3_scale_dedup_one_million_documents():
    """The C3 workload at 1M documents (128 tokens, K = 256, LSH(0.8), 10 % planted near-duplicates) built through
    insert_tokens: labels are a fixed point with labels <= i, equal scipy's components of the GPU's own pairs (with and
    without min_jaccard), and for sampled documents the pairs equal GpuLSH.query filtered to d < i."""
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
    sig = dsk.engine.bulk_signatures_device(tok.view(-1), off, n * t, perms)
    rs = np.random.RandomState(0)
    for thr in (None, 0.8):
        ptr, idx, eq = ix.candidate_pairs(thr)
        assert ptr[-1] > ndup // 4, ptr[-1]
        labels = ix.duplicate_clusters(thr)
        assert np.array_equal(labels[labels], labels) and np.all(labels <= np.arange(n))
        rows = np.repeat(np.arange(n), np.diff(ptr))
        assert np.all(idx < rows)
        assert np.array_equal(labels, _components(n, zip(rows.tolist(), idx.tolist())))
        sample = np.sort(rs.choice(n, 3000, replace=False))
        sample = np.unique(np.concatenate([sample, rows[rs.choice(len(rows), 1000)]]))
        sq = sig[torch.from_numpy(sample).cuda()]
        qptr, qidx = ix.query(sq)
        s_host = sq.cpu().numpy().view(np.uint32)
        for j, i in enumerate(sample.tolist()):
            got = dict(zip(idx[ptr[i]:ptr[i + 1]].tolist(), eq[ptr[i]:ptr[i + 1]].tolist()))
            cand = [d for d in qidx[qptr[j]:qptr[j + 1]].tolist() if d < i]
            if cand:
                crow = sig[torch.tensor(cand, device="cuda")].cpu().numpy().view(np.uint32)
                cnt = (crow == s_host[j][None, :]).sum(axis=1)
            else:
                cnt = np.zeros(0, dtype=np.int64)
            want = {d: int(c) for d, c in zip(cand, cnt) if thr is None or float(c) / float(k) >= thr}
            assert got == want, i
