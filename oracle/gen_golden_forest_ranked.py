"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/forest_ranked.npz from the REAL reference's MinHashLSHForest over
WeightedMinHash and MinHash signatures (WeightedMinHashGenerator.minhash, MinHashLSHForest add / index / query / _query,
WeightedMinHash.jaccard, MinHash.jaccard).

Run where an ekzhu/datasketch checkout exists (it imports the reference from it), after lsh.npz and lsh_topk.npz exist:

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_forest_ranked.py

Weighted configurations, each over integer-frequency vectors with planted near-duplicate groups (a base vector and
variants with a share of the non-zero weights re-drawn), as in gen_golden_lsh_weighted.py:

    w0  sample_size 128, l 8   (k 16)
    w1  sample_size 32,  l 32  (k 1)
    w2  sample_size 16,  l 4   (k 4), weights of about 1e-6, so that t is negative (here for every sample)
    w3  sample_size 30,  l 4   (k 7): l * k = 28 < sample_size, the last two samples are never walked

Unweighted configurations over lsh.npz's 300 signatures, with lsh_topk.npz's 120 held-out signatures as queries:

    u8  num_perm 128, l 8
    u32 num_perm 128, l 32

For each: the queries are held-out vectors (``q``) and the first N_SELF indexed ones (``s``).  Stored, as outputs of the
reference's own API:

    <c>_qset<topk> / <c>_sset<topk>   forest.query(m, topk) for topk in 1, 5, 20, 200, sorted, -1 padded
    <c>_q_k<k>_c<c>_t<j>_idx / _jac   sorted([d for d in forest.query(m, c) if m.jaccard(doc[d]) >= t],
                                             key=lambda d: (-m.jaccard(doc[d]), d))[:k], -1 / -1.0 padded
    <c>_s_k<k>_c<c>_t<j>_idx / _jac   the same ranking over the neighbour candidates of indexed document i:
                                             the first c distinct d != i of the _query loop (r = k..1), stopping as
                                             query stops
for k in 1, 5, 32, c in k, 2k, 100 and t in None, 0.5 (j = 0, 1).  It pins tests/test_lshforest_weighted.py and
tests/test_lshforest_topk.py.
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
from datasketch import MinHash, MinHashLSHForest, WeightedMinHashGenerator  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
#          name  ss  l   dim  bases variants scale
WEIGHTED = (("w0", 128, 8, 96, 30, 5, 1.0),
            ("w1", 32, 32, 64, 30, 5, 1.0),
            ("w2", 16, 4, 40, 30, 5, 1e-6),
            ("w3", 30, 4, 48, 30, 5, 1.0))
UNWEIGHTED = (("u8", 8), ("u32", 32))
QSETS = (1, 5, 20, 200)
KS = (1, 5, 32)
THRESHOLDS = (None, 0.5)
N_SELF = 60


def cands(k):
    return sorted({k, 2 * k, 100})


def _vector(rs, dim):
    v = rs.randint(1, 20, size=dim) * (rs.rand(dim) >= 0.6)
    if not v.any():
        v[rs.randint(dim)] = rs.randint(1, 20)
    return v


def _variant(rs, v, frac):
    w = v.copy()
    nz = np.flatnonzero(w)
    pick = rs.choice(nz, max(1, int(round(frac * len(nz)))), replace=False)
    w[pick] = rs.randint(1, 20, size=len(pick))
    return w


def _pad(xs, width, fill, dtype):
    out = np.full(width, fill, dtype=dtype)
    out[:len(xs)] = xs
    return out


def neighbour_candidates(forest, m, i, c):
    """The reference's walk of query(m, c) (lshforest.py:92-128) with document i left out."""
    res = set()
    for r in range(forest.k, 0, -1):
        for d in forest._query(m, r, forest.l):
            if d != i:
                res.add(d)
            if len(res) >= c:
                return res
    return res


def ranked(m, cand, ms, k, t):
    keep = [d for d in cand if t is None or m.jaccard(ms[d]) >= t]
    best = sorted(keep, key=lambda d: (-m.jaccard(ms[d]), d))[:k]
    return _pad(best, k, -1, np.int32), _pad([m.jaccard(ms[d]) for d in best], k, -1.0, np.float64)


def gen_forest(name, ms, qs, l):
    forest = MinHashLSHForest(num_perm=len(ms[0]), l=l)
    for i, m in enumerate(ms):
        forest.add(i, m)
    forest.index()
    d = {}
    selfq = ms[:N_SELF]
    for topk in QSETS:
        d["qset%d" % topk] = np.stack([_pad(sorted(forest.query(m, topk)), topk, -1, np.int32) for m in qs])
        d["sset%d" % topk] = np.stack([_pad(sorted(forest.query(m, topk)), topk, -1, np.int32) for m in selfq])
    for k in KS:
        for c in cands(k):
            qc = [forest.query(m, c) for m in qs]
            sc = [neighbour_candidates(forest, m, i, c) for i, m in enumerate(selfq)]
            for j, t in enumerate(THRESHOLDS):
                for tag, queries, cs in (("q", qs, qc), ("s", selfq, sc)):
                    rows = [ranked(m, x, ms, k, t) for m, x in zip(queries, cs)]
                    d["%s_k%d_c%d_t%d_idx" % (tag, k, c, j)] = np.stack([x[0] for x in rows])
                    d["%s_k%d_c%d_t%d_jac" % (tag, k, c, j)] = np.stack([x[1] for x in rows])
    return {name + "_" + key: v for key, v in d.items()}


def gen_weighted(name, ss, l, dim, bases, variants, scale, rs):
    X = []
    for _ in range(bases):
        v = _vector(rs, dim)
        X.append(v)
        for j in range(variants - 1):
            X.append(_variant(rs, v, (0.05, 0.1, 0.2, 0.3)[j % 4]))
    X = np.stack(X)[rs.permutation(bases * variants)]
    n = len(X)
    qX = np.stack([_variant(rs, X[i], (0.05, 0.1, 0.2)[j % 3]) for j, i in enumerate(rs.choice(n, 20, replace=False))]
                  + [X[i].copy() for i in rs.choice(n, 10, replace=False)]
                  + [_vector(rs, dim) for _ in range(10)])
    qX = qX[rs.permutation(len(qX))]
    X, qX = X * scale, qX * scale
    mg = WeightedMinHashGenerator(dim, sample_size=ss, seed=1)
    ms = [mg.minhash(v.astype(np.float64)) for v in X]
    qs = [mg.minhash(v.astype(np.float64)) for v in qX]
    d = gen_forest(name, ms, qs, l)
    d[name + "_params"] = np.array([ss, l, 1], dtype=np.int64)
    d[name + "_X"] = X.astype(np.float64)
    d[name + "_hv"] = np.stack([m.hashvalues for m in ms]).astype(np.int64)
    d[name + "_qX"] = qX.astype(np.float64)
    d[name + "_qhv"] = np.stack([m.hashvalues for m in qs]).astype(np.int64)
    return d


def gen_unweighted(name, l):
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    qsig = np.load(os.path.join(OUT, "lsh_topk.npz"))["qsig"]
    ms = [MinHash(num_perm=128, hashvalues=row.astype(np.uint64)) for row in sig]
    qs = [MinHash(num_perm=128, hashvalues=row.astype(np.uint64)) for row in qsig]
    d = gen_forest(name, ms, qs, l)
    d[name + "_params"] = np.array([128, l, 0], dtype=np.int64)
    return d


def gen_forest_ranked():
    rs = np.random.RandomState(83)
    d = {"ks": np.array(KS, dtype=np.int64), "qsets": np.array(QSETS, dtype=np.int64),
         "thresholds": np.array([-1.0 if t is None else t for t in THRESHOLDS], dtype=np.float64),
         "n_self": np.array(N_SELF, dtype=np.int64)}
    for cfg in WEIGHTED:
        d.update(gen_weighted(*cfg, rs))
    for cfg in UNWEIGHTED:
        d.update(gen_unweighted(*cfg))
    np.savez_compressed(os.path.join(OUT, "forest_ranked.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_forest_ranked()
    print("forest_ranked.npz", os.path.getsize(os.path.join(OUT, "forest_ranked.npz")))
