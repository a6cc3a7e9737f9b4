"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/*.npz from the REAL reference.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden.py [fixture ...]

With fixture names (``wmh_special``, ``lsh``, ...) only those files are written.

Every array written here is an output of the unmodified reference's public API
(``MinHash``, ``LeanMinHash``, ``WeightedMinHashGenerator``, ``MinHashLSH``) on
the seeded inputs stored next to it, so the fixtures pin both the oracle
(oracle/oracle_np.py, oracle/oracle_c.c) and the CUDA path.
"""
from __future__ import annotations

import os
import sys

import numpy as np

REF = os.environ["DATASKETCH_REF"]
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import fake_backends  # noqa: E402  in-memory stand-ins for the optional `redis` / `pybloomfilter` packages
fake_backends.install()           # must precede the import below: storage.py / lsh_bloom.py probe them at import time
import datasketch  # noqa: E402  (the reference)
from datasketch import LeanMinHash, MinHash, MinHashLSH, WeightedMinHashGenerator  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def ident(x):
    return int(x)


def ragged(rs, n, maxlen, hi=2 ** 32, dtype=np.uint64):
    lens = rs.randint(0, maxlen + 1, size=n)
    lens[:3] = [0, 1, 2]            # empty / single / pair documents
    lens[-1] = 0                    # trailing empty document
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = rs.randint(0, hi, size=int(off[-1]), dtype=dtype)
    return tok, off


def ref_bulk(tok, off, **kw):
    docs = [[int(x) for x in tok[off[i]:off[i + 1]]] for i in range(len(off) - 1)]
    ms = MinHash.bulk(docs, hashfunc=ident, **kw)
    return np.stack([m.hashvalues for m in ms]) if ms else np.zeros((0, kw["num_perm"]), np.uint64)


def gen_minhash():
    d = {}
    # the reference's own absolute golden (test/test_minhash.py:109-115)
    m = MinHash(4, 1)
    m.update(b"Hello")
    d["hello_k4_seed1"] = m.hashvalues.copy()
    # permutations (minhash.py:170-184)
    for k, seed in [(4, 1), (128, 1), (256, 7), (100, 42)]:
        d[f"perm_k{k}_s{seed}"] = MinHash(num_perm=k, seed=seed).permutations
    # C1: 1000 docs x 64 tokens, K=128, seed=1 (BASELINE.json configs[0])
    rs = np.random.RandomState(0)
    tok = rs.randint(0, 2 ** 32, size=(1000, 64), dtype=np.uint64)
    d["c1_tokens"] = tok.astype(np.uint32)
    off = np.arange(1001, dtype=np.int64) * 64
    sig = ref_bulk(tok.reshape(-1), off, num_perm=128, seed=1)
    assert sig.max() < 2 ** 32
    d["c1_sig"] = sig.astype(np.uint32)
    # ragged batches incl. empty docs, several K / seeds
    for k, seed in [(4, 1), (100, 42), (128, 1), (256, 7), (33, 5)]:
        rs = np.random.RandomState(100 + k)
        tok, off = ragged(rs, 120, 300)
        d[f"rag_k{k}_tokens"] = tok.astype(np.uint32)
        d[f"rag_k{k}_offsets"] = off
        d[f"rag_k{k}_seed"] = np.int64(seed)
        d[f"rag_k{k}_sig"] = ref_bulk(tok, off, num_perm=k, seed=seed).astype(np.uint32)
    # a long document (T >> K) and tiny-hash tokens (small ints as in test/utils.py fake_hash_func)
    rs = np.random.RandomState(7)
    tok = rs.randint(0, 2 ** 32, size=20000, dtype=np.uint64)
    off = np.array([0, 20000], dtype=np.int64)
    d["long_tokens"] = tok.astype(np.uint32)
    d["long_sig"] = ref_bulk(tok, off, num_perm=128, seed=1).astype(np.uint32)
    small = np.arange(0, 64, dtype=np.uint64) * 4
    d["small_tokens"] = small.astype(np.uint32)
    d["small_sig"] = ref_bulk(small, np.array([0, 64], np.int64), num_perm=128, seed=1).astype(np.uint32)
    # default SHA1 hashfunc on byte tokens (test/test_minhash_gpu.py:20-52 shapes)
    data = [f"token-{i}".encode("utf-8") for i in range(1000)]
    m = MinHash(num_perm=256, seed=7)
    m.update_batch(data)
    d["sha1_k256_s7_n1000"] = m.hashvalues.copy()
    m = MinHash(num_perm=128, seed=7)
    m.update_batch(data[:500])
    m.update_batch([f"token-{i}".encode("utf-8") for i in range(700)])
    d["sha1_k128_s7_500_700"] = m.hashvalues.copy()
    # hash values wider than 32 bits (minhash.py:294 casts to uint64)
    rs = np.random.RandomState(11)
    tok, off = ragged(rs, 40, 50, hi=2 ** 63, dtype=np.uint64)
    tok[::3] |= np.uint64(1) << np.uint64(63)
    tok[1::5] = rs.randint(2 ** 32, 2 ** 40, size=len(tok[1::5]), dtype=np.uint64)
    d["u64_tokens"] = tok
    d["u64_offsets"] = off
    d["u64_sig"] = ref_bulk(tok, off, num_perm=64, seed=3)
    # update_batch on a non-empty state, then jaccard / merge / union
    m1 = MinHash(num_perm=128, seed=1, hashfunc=ident)
    m1.update_batch(range(0, 300))
    m2 = MinHash(num_perm=128, seed=1, hashfunc=ident)
    m2.update_batch(range(150, 450))
    d["j_m1"], d["j_m2"] = m1.hashvalues.copy(), m2.hashvalues.copy()
    d["j_jaccard"] = np.float64(m1.jaccard(m2))
    d["j_count1"] = np.float64(m1.count())
    mm = m1.copy()
    mm.merge(m2)
    d["j_merge"] = mm.hashvalues.copy()
    d["j_union"] = MinHash.union(m1, m2).hashvalues.copy()
    np.savez_compressed(os.path.join(OUT, "minhash.npz"), **d)


def gen_lean():
    d = {}
    m = MinHash(10, 1, hashfunc=ident)
    m.update(123)
    lm = LeanMinHash(m)
    d["hashvalues"] = lm.hashvalues.copy()
    d["seed"] = np.int64(lm.seed)
    names = {"@": "native", "=": "std", "<": "le", ">": "be", "!": "net"}
    for bo, nm in names.items():
        buf = bytearray(lm.bytesize(bo))
        lm.serialize(buf, bo)
        d[f"buf_{nm}"] = np.frombuffer(bytes(buf), dtype=np.uint8)
        d[f"size_{nm}"] = np.int64(lm.bytesize(bo))
    d["getstate"] = np.frombuffer(bytes(lm.__getstate__()), dtype=np.uint8)
    d["pyhash"] = np.int64(hash(lm))
    # a batch: C1-like signatures -> records
    rs = np.random.RandomState(5)
    sig = rs.randint(0, 2 ** 32, size=(16, 128), dtype=np.uint64)
    recs = []
    for row in sig:
        l = LeanMinHash(seed=9, hashvalues=row)
        buf = bytearray(l.bytesize())
        l.serialize(buf)
        recs.append(np.frombuffer(bytes(buf), dtype=np.uint8))
    d["batch_sig"] = sig.astype(np.uint32)
    d["batch_recs"] = np.stack(recs)
    np.savez_compressed(os.path.join(OUT, "lean.npz"), **d)


def gen_wmh():
    d = {}
    for dim, ss, seed, nvec, tag in [(64, 16, 1, 24, "small"), (4096, 128, 1, 3, "c4"), (5, 8, 3, 6, "tiny")]:
        g = WeightedMinHashGenerator(dim, ss, seed)
        rs = np.random.RandomState(4)
        v = rs.uniform(0, 10, (nvec, dim)).astype(np.float32)
        v[:, ::7] = 0
        if tag == "small":
            v[1] = np.floor(v[1])            # integer frequencies incl. extra zeros
            v[2, 2:] = 0                     # single non-zero (col 1)
            v[3] *= 1e-6                     # tiny weights -> negative logs
            v[4] *= 1e6
        out = np.stack([g.minhash(x).hashvalues for x in v]).astype(np.int64)
        d[f"{tag}_v"] = v
        d[f"{tag}_out"] = out
        d[f"{tag}_cfg"] = np.array([dim, ss, seed], dtype=np.int64)
        if tag != "c4":
            d[f"{tag}_rs"], d[f"{tag}_ln_cs"], d[f"{tag}_betas"] = g.rs, g.ln_cs, g.betas
        else:  # params are 6 MB; pin them by a few samples + sums
            d["c4_rs_head"], d["c4_ln_cs_head"], d["c4_betas_head"] = g.rs[:2, :64], g.ln_cs[:2, :64], g.betas[:2, :64]
            d["c4_sums"] = np.array([g.rs.astype(np.float64).sum(), g.ln_cs.astype(np.float64).sum(),
                                     g.betas.astype(np.float64).sum()])
    np.savez_compressed(os.path.join(OUT, "wmh.npz"), **d)


def gen_wmh_many():
    """WeightedMinHashGenerator.minhash_many (weighted_minhash.py:161-247), dense and scipy.sparse input,
    with all-zero rows (-> None)."""
    import scipy.sparse
    d = {}
    for dim, ss, seed, nvec, tag in [(64, 16, 1, 40, "small"), (5, 8, 3, 9, "tiny"), (300, 32, 7, 25, "mid")]:
        g = WeightedMinHashGenerator(dim, ss, seed)
        rs = np.random.RandomState(14)
        X = np.floor(rs.uniform(0, 6, (nvec, dim))).astype(np.float32)   # integer frequencies, many zeros
        X[rs.uniform(size=X.shape) < 0.5] = 0
        X[3] = 0
        X[nvec - 1] = 0
        X[5] = rs.uniform(0, 1e-3, dim)                                   # tiny weights: negative logs
        dense = g.minhash_many(X)
        sparse = g.minhash_many(scipy.sparse.csr_matrix(X))
        null = np.array([m is None for m in dense])
        assert (null == np.array([m is None for m in sparse])).all() and null[3] and null[nvec - 1]
        out = np.zeros((nvec, ss, 2), dtype=np.int64)
        for i, (a, b) in enumerate(zip(dense, sparse)):
            if a is not None:
                assert np.array_equal(a.hashvalues, b.hashvalues)
                out[i] = a.hashvalues
        d[f"{tag}_X"], d[f"{tag}_out"], d[f"{tag}_null"] = X, out, null
        d[f"{tag}_cfg"] = np.array([dim, ss, seed], dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "wmh_many.npz"), **d)


WMH_SPECIAL_ROWS = [                               # dim 6: zero / -0.0 / negative / NaN / +-inf / subnormal / FLT_MAX
    [1, 2, np.inf, 4, 0, 5],
    [1, 2, -3, 4, 0, 5],
    [1, 2, np.nan, 4, 0, 5],
    [-1, -2, 0, 0, 0, 0],                          # all negative
    [np.nan, np.nan, 0, 0, 0, np.nan],             # all NaN
    [0, 0, 0, 0, 0, 0],                            # all zero
    [-0.0, 1, 0, 2, -0.0, 3],
    [1e-45, 1e-40, 1, 0, 3.4028235e38, 2],         # subnormals and FLT_MAX
    [0, 0, 0, 0, 0, 1e-45],
    [3.4028235e38, 0, 0, 0, 0, 0],
    [-np.inf, 1, 2, 0, 3, 4],
    [2, np.inf, 1, np.inf, 0, 3],                  # the first +inf wins
    [1, np.nan, -1, 2, 0, np.inf],                 # NaN before a negative weight and +inf
    [0, -5, 1, 1, np.inf, np.nan],
    [1, 1, 1, 1, 1, 1],
]


def gen_wmh_special():
    """WeightedMinHashGenerator.minhash (values, or the exception's type name) and minhash_many on rows holding zeros,
    -0.0, negative, NaN, +-inf, subnormal and FLT_MAX weights, for two (sample_size, seed) choices."""
    import warnings
    d = {}
    X = np.array(WMH_SPECIAL_ROWS, dtype=np.float32)
    for dim, ss, seed, tag in [(6, 4, 1, "a"), (6, 16, 5, "b")]:
        g = WeightedMinHashGenerator(dim, ss, seed)
        out = np.zeros((len(X), ss, 2), dtype=np.int64)
        err = []
        for i, v in enumerate(X):
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    out[i] = g.minhash(v).hashvalues
                err.append("")
            except Exception as e:  # noqa: BLE001  (the exception type is the expected value)
                err.append(type(e).__name__)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            many = g.minhash_many(X)
        many_out = np.zeros((len(X), ss, 2), dtype=np.int64)
        for i, m in enumerate(many):
            if m is not None:
                many_out[i] = m.hashvalues
        d[f"{tag}_cfg"] = np.array([dim, ss, seed], dtype=np.int64)
        d[f"{tag}_out"], d[f"{tag}_err"] = out, np.array(err)
        d[f"{tag}_many_out"], d[f"{tag}_many_null"] = many_out, np.array([m is None for m in many])
    d["X"] = X
    np.savez_compressed(os.path.join(OUT, "wmh_special.npz"), **d)


def gen_ensemble():
    """MinHashLSHEnsemble (lshensemble.py, lshensemble_partition.py): parameter tables, partition bounds and the
    query results of a small indexed corpus."""
    from datasketch.lshensemble import MinHashLSHEnsemble
    from datasketch.lshensemble_partition import optimal_partitions
    d = {}
    rs = np.random.RandomState(31)
    # partition bounds on a few size distributions (incl. num_part 1, 2, > domain)
    cases = []
    for n, num_part in [(1, 4), (5, 1), (6, 2), (9, 3), (12, 5), (20, 8), (30, 16), (7, 7), (7, 9)]:
        sizes = np.sort(rs.choice(np.arange(1, 500), size=n, replace=False)).astype(np.int64)
        counts = rs.randint(1, 30, size=n).astype(np.int64)
        b = np.array(optimal_partitions(sizes, counts, num_part), dtype=np.int64)
        cases.append((sizes, counts, num_part, b))
    for i, (sizes, counts, num_part, b) in enumerate(cases):
        d[f"part{i}_sizes"], d[f"part{i}_counts"], d[f"part{i}_bounds"] = sizes, counts, b
        d[f"part{i}_num_part"] = np.array([num_part], dtype=np.int64)
    d["n_part_cases"] = np.array([len(cases)], dtype=np.int64)
    # parameter tables
    for i, (thr, k, m, w) in enumerate([(0.5, 32, 4, (0.5, 0.5)), (0.8, 32, 8, (0.5, 0.5)), (0.2, 16, 4, (0.3, 0.7))]):
        e = MinHashLSHEnsemble(threshold=thr, num_perm=k, num_part=2, m=m, weights=w)
        d[f"par{i}_cfg"] = np.array([thr, k, m, w[0], w[1]], dtype=np.float64)
        d[f"par{i}_params"], d[f"par{i}_xqs"] = e.params.astype(np.int64), e.xqs
    # end to end: sets of very different sizes drawn from one vocabulary; queries are subsets of indexed sets
    k = 32
    vocab = rs.randint(0, 2 ** 32, size=3000, dtype=np.uint64)
    sets = []
    for i in range(160):
        size = int(rs.choice([5, 8, 13, 20, 40, 80, 150, 300, 600]))
        sets.append(rs.choice(vocab, size=size, replace=False))
    for i in range(0, 160, 4):                      # containment pairs: sets[i] is a subset of sets[i+1]
        big = sets[i + 1]
        sets[i] = rs.choice(big, size=max(3, len(big) // 3), replace=False)
    mhs = MinHash.bulk([[int(t) for t in s] for s in sets], num_perm=k, seed=1, hashfunc=ident)
    sig = np.stack([m.hashvalues for m in mhs])
    sizes = np.array([len(s) for s in sets], dtype=np.int64)
    ens = MinHashLSHEnsemble(threshold=0.5, num_perm=k, num_part=6, m=4)
    ens.index([(i, mhs[i], int(sizes[i])) for i in range(len(sets))])
    d["e2e_sig"], d["e2e_sizes"] = sig.astype(np.uint32), sizes
    d["e2e_cfg"] = np.array([0.5, k, 6, 4], dtype=np.float64)
    d["e2e_lowers"] = np.array([-1 if x is None else x for x in ens.lowers], dtype=np.int64)
    d["e2e_uppers"] = np.array([-1 if x is None else x for x in ens.uppers], dtype=np.int64)
    qptr, qidx = [0], []
    for i in range(len(sets)):
        res = sorted(set(ens.query(mhs[i], int(sizes[i]))))
        qidx.extend(res)
        qptr.append(len(qidx))
    d["e2e_qptr"], d["e2e_qidx"] = np.array(qptr, dtype=np.int64), np.array(qidx, dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "ensemble.npz"), **d)


def gen_hashes():
    """Token-hash fixtures from the third-party packages the reference's docs name (docs/minhash.rst:79-112).
    Only `xxhash` is installed in the build container; MurmurHash3 is pinned by published vectors in the tests."""
    import xxhash
    rs = np.random.RandomState(77)
    toks = [b"", b"a", b"abc", b"Hello", b"x" * 15, b"y" * 16, b"z" * 17, b"w" * 31, b"v" * 32, b"u" * 33] + \
           [bytes(rs.randint(0, 256, size=rs.randint(0, 120)).astype(np.uint8)) for _ in range(400)]
    blob = np.frombuffer(b"".join(toks), dtype=np.uint8)
    off = np.zeros(len(toks) + 1, dtype=np.int64)
    np.cumsum([len(t) for t in toks], out=off[1:])
    d = {"blob": blob, "off": off, "xxhash_version": np.array([xxhash.VERSION])}
    for seed in (0, 1, 0x9747B28C):
        d[f"xxh32_seed{seed}"] = np.array([xxhash.xxh32_intdigest(t, seed) for t in toks], dtype=np.uint32)
    np.savez_compressed(os.path.join(OUT, "hashes.npz"), **d)


def gen_lsh():
    d = {}
    rows = []
    for thr, k, w in [(0.5, 128, (0.5, 0.5)), (0.8, 128, (0.5, 0.5)), (0.9, 128, (0.5, 0.5)),
                      (0.8, 256, (0.5, 0.5)), (0.8, 128, (0.2, 0.8)), (0.5, 16, (0.5, 0.5)), (0.5, 32, (0.5, 0.5))]:
        l = MinHashLSH(threshold=thr, num_perm=k, weights=w)
        rows.append([thr, k, w[0], w[1], l.b, l.r])
    d["params"] = np.array(rows, dtype=np.float64)
    # band keys of a few signatures (lsh.py:344, :537-538)
    rs = np.random.RandomState(21)
    docs = [rs.randint(0, 2 ** 32, size=rs.randint(20, 80), dtype=np.uint64) for _ in range(300)]
    # plant near-duplicates so buckets are non-trivial
    for i in range(0, 300, 3):
        src = docs[i].copy()
        nres = max(1, len(src) // 12)
        src[rs.choice(len(src), nres, replace=False)] = rs.randint(0, 2 ** 32, size=nres, dtype=np.uint64)
        docs[i + 1] = src
        docs[i + 2] = docs[i].copy()     # exact duplicate
    ms = MinHash.bulk([[int(t) for t in doc] for doc in docs], num_perm=128, seed=1, hashfunc=ident)
    sig = np.stack([m.hashvalues for m in ms])
    d["sig"] = sig.astype(np.uint32)
    lsh = MinHashLSH(threshold=0.8, num_perm=128)
    d["b_r"] = np.array([lsh.b, lsh.r], dtype=np.int64)
    for i, m in enumerate(ms):
        lsh.insert(i, m)
    keys0 = lsh.keys[0]
    d["keys_doc0"] = np.frombuffer(b"".join(keys0), dtype=np.uint8).reshape(lsh.b, 8 * lsh.r)
    res, ptr = [], [0]
    for m in ms:
        r = sorted(lsh.query(m))
        res.extend(r)
        ptr.append(len(res))
    d["query_idx"] = np.array(res, dtype=np.int64)
    d["query_ptr"] = np.array(ptr, dtype=np.int64)
    counts = lsh.get_counts()
    d["bucket_counts_sorted"] = np.array(sorted(c for t in counts for c in t.values()), dtype=np.int64)
    # the reference's pinned candidate set (test/test_lsh.py:109-125): {0, 1}
    l2 = MinHashLSH(threshold=0.5, num_perm=32)
    mh = []
    for toks in ([b"a", b"b", b"c"], [b"a", b"b", b"d"], [b"x", b"y", b"z"]):
        m = MinHash(num_perm=32)
        for t in toks:
            m.update(t)
        mh.append(m)
    for i, m in enumerate(mh):
        l2.insert(i, m)
    d["abc_sig"] = np.stack([m.hashvalues for m in mh])
    d["abc_query0"] = np.array(sorted(l2.query(mh[0])), dtype=np.int64)
    d["abc_b_r"] = np.array([l2.b, l2.r], dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "lsh.npz"), **d)


def gen_bbit():
    from datasketch.b_bit_minhash import bBitMinHash
    d = {}
    m = MinHash(num_perm=128, seed=1, hashfunc=ident)
    for v in (11, 123, 92, 98, 123218, 32):
        m.update(v)
    m2 = MinHash(num_perm=128, seed=1, hashfunc=ident)
    for v in (11, 123, 92, 98, 7, 32):
        m2.update(v)
    d["hv1"], d["hv2"] = m.hashvalues.copy(), m2.hashvalues.copy()
    bs = [1, 2, 3, 4, 5, 8, 12, 16, 27, 32]
    d["bs"] = np.array(bs, dtype=np.int64)
    for b in bs:
        x, y = bBitMinHash(m, b), bBitMinHash(m2, b)
        d[f"state_b{b}"] = np.frombuffer(bytes(x.__getstate__()), dtype=np.uint8)
        d[f"hv_b{b}"] = x.hashvalues.copy()
        d[f"jac_b{b}"] = np.float64(x.jaccard(y))
        d[f"size_b{b}"] = np.int64(x.bytesize())
    xr, yr = bBitMinHash(m, 4, r=0.3), bBitMinHash(m2, 4, r=0.1)
    d["jac_b4_r"] = np.float64(xr.jaccard(yr))
    np.savez_compressed(os.path.join(OUT, "bbit.npz"), **d)


def gen_forest():
    """MinHashLSHForest.query results (as sorted id lists) on the lsh.npz signatures, several (l, k)."""
    from datasketch import MinHashLSHForest
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    d = {}
    for l in (8, 32):
        f = MinHashLSHForest(num_perm=128, l=l)
        for i, row in enumerate(sig):
            f.add(i, LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)))
        f.index()
        for topk in (1, 5, 20):
            res, ptr = [], [0]
            for row in sig[:120]:
                r = sorted(f.query(LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)), topk))
                res.extend(r)
                ptr.append(len(res))
            d[f"l{l}_k{topk}_idx"] = np.array(res, dtype=np.int64)
            d[f"l{l}_k{topk}_ptr"] = np.array(ptr, dtype=np.int64)
        if l == 8:
            d["keys_doc0"] = np.frombuffer(b"".join(f.keys[0]), dtype=np.uint8)
            d["hashvalues_doc3"] = f.get_minhash_hashvalues(3)
    np.savez_compressed(os.path.join(OUT, "forest.npz"), **d)


def gen_bloom():
    """MinHashLSHBloom (lsh_bloom.py) run on the pybloomfilter stand-in: the values BloomTable.insert hands to the filter
    ARE the band keys `sum(hashvalues) % _mersenne_prime` (:105); query answers with exact-membership tables."""
    import warnings
    from datasketch.lsh_bloom import MinHashLSHBloom
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    d = {}
    rows = []
    for thr, k in [(0.5, 128), (0.8, 128), (0.9, 128), (0.5, 32)]:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            l = MinHashLSHBloom(threshold=thr, num_perm=k, n=100, fp=0.01)
        rows.append([thr, k, l.b, l.r])
    d["params"] = np.array(rows, dtype=np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        bl = MinHashLSHBloom(threshold=0.8, num_perm=128, n=1000, fp=0.001)
    d["b_r"] = np.array([bl.b, bl.r], dtype=np.int64)
    fake_backends.reset()
    n_ins = 200
    for row in sig[:n_ins]:
        bl.insert(LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)))
    d["keys_inserted"] = np.array([v for _, v in fake_backends.BLOOM_ADDS], dtype=np.uint64).reshape(n_ins, bl.b)
    d["query_all"] = np.array([bl.query(LeanMinHash(seed=1, hashvalues=row.astype(np.uint64))) for row in sig], dtype=np.bool_)
    np.savez_compressed(os.path.join(OUT, "bloom.npz"), **d)


def gen_storage():
    """MinHashLSH over the reference's Redis storage (storage.py:819-1049) on the redis stand-in: the database state
    after the inserts, i.e. the wire layout an existing deployment reads (lsh.py:191-200)."""
    import pickle
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    d = {}
    cases = {"pickled": dict(prepickle=None, keys=[("doc", i) for i in range(120)]),
             "bytes": dict(prepickle=False, keys=[b"k%04d" % i for i in range(120)])}
    for name, c in cases.items():
        fake_backends.reset()
        lsh = MinHashLSH(threshold=0.8, num_perm=128, prepickle=c["prepickle"],
                         storage_config={"type": "redis", "basename": b"gpuidx", "redis": {"host": "nowhere", "port": 0}})
        for key, row in zip(c["keys"], sig):
            lsh.insert(key, LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)))
        state = {"hash": {k: dict(v) for k, v in fake_backends.DB["hash"].items()},
                 "list": {k: list(v) for k, v in fake_backends.DB["list"].items()},
                 "set": {k: sorted(v) for k, v in fake_backends.DB["set"].items()}}
        d[name + "_state"] = np.frombuffer(pickle.dumps(state, protocol=4), dtype=np.uint8)
        d[name + "_b_r"] = np.array([lsh.b, lsh.r], dtype=np.int64)
        q = sorted(lsh.query(LeanMinHash(seed=1, hashvalues=sig[0].astype(np.uint64))), key=repr)
        d[name + "_query0"] = np.frombuffer(pickle.dumps(q, protocol=4), dtype=np.uint8)
    np.savez_compressed(os.path.join(OUT, "storage.npz"), **d)


def gen_storage_cassandra():
    """MinHashLSH over the reference's Cassandra storage (storage.py:262-819) on the cassandra-driver stand-in: the rows
    of every table in the order they were written (ts), the DDL, and a query answered from those rows."""
    import pickle
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    d = {}
    cases = {"pickled": dict(prepickle=True, keys=[("doc", i) for i in range(120)]),
             "bytes": dict(prepickle=None, keys=[b"k%04d" % i for i in range(120)])}
    for name, c in cases.items():
        fake_backends.reset()
        cfg = {"type": "cassandra", "basename": b"gpuidx",
               "cassandra": {"seeds": ["nowhere"], "keyspace": "lsh_test",
                             "replication": {"class": "SimpleStrategy", "replication_factor": "1"},
                             "drop_keyspace": False, "drop_tables": False}}
        lsh = MinHashLSH(threshold=0.8, num_perm=128, prepickle=c["prepickle"], storage_config=cfg)
        for key, row in zip(c["keys"], sig):
            lsh.insert(key, LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)))
        state = {t: [kv for kv, _ in sorted(rows.items(), key=lambda x: x[1])] for t, rows in fake_backends.CQL["tables"].items()}
        d[name + "_state"] = np.frombuffer(pickle.dumps(state, protocol=4), dtype=np.uint8)
        d[name + "_ddl"] = np.frombuffer(pickle.dumps([q for q in fake_backends.CQL["ddl"] if q.startswith("CREATE TABLE")],
                                                      protocol=4), dtype=np.uint8)
        d[name + "_b_r"] = np.array([lsh.b, lsh.r], dtype=np.int64)
        q = sorted(lsh.query(LeanMinHash(seed=1, hashvalues=sig[0].astype(np.uint64))), key=repr)
        d[name + "_query0"] = np.frombuffer(pickle.dumps(q, protocol=4), dtype=np.uint8)
    np.savez_compressed(os.path.join(OUT, "storage_cassandra.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gens = {"minhash": gen_minhash, "lean": gen_lean, "wmh": gen_wmh, "wmh_many": gen_wmh_many,
            "wmh_special": gen_wmh_special, "lsh": gen_lsh, "bbit": gen_bbit, "forest": gen_forest,
            "ensemble": gen_ensemble, "hashes": gen_hashes, "bloom": gen_bloom, "storage": gen_storage,
            "storage_cassandra": gen_storage_cassandra}
    for name in sys.argv[1:] or gens:
        gens[name]()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))
