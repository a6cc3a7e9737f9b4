"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_weighted.npz from the REAL reference's MinHashLSH over
WeightedMinHash signatures (WeightedMinHashGenerator.minhash, MinHashLSH insert / query / remove, WeightedMinHash.jaccard).

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_weighted.py

Three configurations, each over integer-frequency vectors (about 60 % zeros) with planted near-duplicate groups: a base
vector and variants of it in which a share of the non-zero weights is re-drawn.

    a   sample_size 32,  dim 64,  MinHashLSH(threshold=0.5)
    b   sample_size 128, dim 128, MinHashLSH(params=(40, 3)): more than 32 bands
    c   sample_size 4,   dim 10,  MinHashLSH(threshold=0.5), the size of the reference's own TestWeightedMinHashLSH

For each, with keys 0..N-1 = the indexed vectors' numbers, the file stores the vectors and the reference's hashvalues, the
query lists (CSR, sorted) of held-out vectors (``q``) and of indexed vectors (``s``), the WeightedMinHash.jaccard of every
(query, candidate), the lists filtered at two thresholds, the streaming dedup loop over the held-out batch

    for m in batch:
        if not [d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]:
            lsh.insert(len(doc), m)

(kept mask, the kept-or-indexed candidate with the largest jaccard, smallest key among equal ones, and that jaccard) at
both thresholds, and the query lists after removing 20 keys.  It pins tests/test_lsh_weighted.py's oracle and the CUDA path.
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
from datasketch import MinHashLSH, WeightedMinHashGenerator  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
#       name  ss   dim  threshold params    bases variants thresholds
CONFIGS = (("a", 32, 64, 0.5, None, 30, 5, (0.5, 0.75)),
           ("b", 128, 128, 0.9, (40, 3), 30, 5, (0.6, 0.85)),
           ("c", 4, 10, 0.5, None, 12, 5, (0.5, 1.0)))
N_SELF, N_REMOVED = 30, 20


def _vector(rs, dim):
    v = rs.randint(1, 20, size=dim) * (rs.rand(dim) >= 0.6)
    if not v.any():
        v[rs.randint(dim)] = rs.randint(1, 20)
    return v


def _variant(rs, v, frac):
    """A share ``frac`` of v's non-zero weights re-drawn (at least one)."""
    w = v.copy()
    nz = np.flatnonzero(w)
    pick = rs.choice(nz, max(1, int(round(frac * len(nz)))), replace=False)
    w[pick] = rs.randint(1, 20, size=len(pick))
    return w


def _csr(lists):
    ptr = np.zeros(len(lists) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(x) for x in lists])
    idx = np.array([d for x in lists for d in x], dtype=np.int64)
    return ptr, idx


def gen_config(name, ss, dim, threshold, params, bases, variants, thresholds, rs):
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
    mg = WeightedMinHashGenerator(dim, sample_size=ss, seed=1)
    ms = [mg.minhash(v.astype(np.float64)) for v in X]
    qs = [mg.minhash(v.astype(np.float64)) for v in qX]

    def fresh():
        lsh = MinHashLSH(threshold=threshold, num_perm=ss, params=params)
        for i, m in enumerate(ms):
            lsh.insert(i, m)
        return lsh

    lsh = fresh()
    d = {"params": np.array([lsh.b, lsh.r, ss], dtype=np.int64),
         "thresholds": np.array(thresholds, dtype=np.float64),
         "X": X.astype(np.float32), "hv": np.stack([m.hashvalues for m in ms]).astype(np.int64),
         "qX": qX.astype(np.float32), "qhv": np.stack([m.hashvalues for m in qs]).astype(np.int64)}
    for tag, queries in (("q", qs), ("s", ms[:N_SELF])):
        lists = [sorted(lsh.query(m)) for m in queries]
        d[tag + "_ptr"], d[tag + "_idx"] = _csr(lists)
        d[tag + "_jaccard"] = np.array([m.jaccard(ms[c]) for m, x in zip(queries, lists) for c in x], dtype=np.float64)
        for j, t in enumerate(thresholds):
            d["%s_kept%d_ptr" % (tag, j)], d["%s_kept%d_idx" % (tag, j)] = _csr(
                [[c for c in x if m.jaccard(ms[c]) >= t] for m, x in zip(queries, lists)])
    for j, t in enumerate(thresholds):
        lsh = fresh()
        held = dict(enumerate(ms))
        kept, match, jac = [], [], []
        for m in qs:
            cand = [c for c in lsh.query(m) if m.jaccard(held[c]) >= t]
            if cand:
                best = min(cand, key=lambda c: (-m.jaccard(held[c]), c))
                kept.append(False)
                match.append(best)
                jac.append(m.jaccard(held[best]))
            else:
                key = len(held)
                lsh.insert(key, m)
                held[key] = m
                kept.append(True)
                match.append(-1)
                jac.append(-1.0)
        d["uniq%d_kept" % j] = np.array(kept, dtype=np.int8)
        d["uniq%d_match" % j] = np.array(match, dtype=np.int64)
        d["uniq%d_jaccard" % j] = np.array(jac, dtype=np.float64)
    lsh = fresh()
    removed = rs.choice(n, N_REMOVED, replace=False)
    for key in removed.tolist():
        lsh.remove(key)
    d["removed"] = removed.astype(np.int64)
    d["rq_ptr"], d["rq_idx"] = _csr([sorted(lsh.query(m)) for m in qs])
    d["rs_ptr"], d["rs_idx"] = _csr([sorted(lsh.query(m)) for m in ms[:N_SELF]])
    return {name + "_" + k: v for k, v in d.items()}


def gen_lsh_weighted():
    rs = np.random.RandomState(61)
    d = {}
    for cfg in CONFIGS:
        d.update(gen_config(*cfg, rs))
    np.savez_compressed(os.path.join(OUT, "lsh_weighted.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_lsh_weighted()
    print("lsh_weighted.npz", os.path.getsize(os.path.join(OUT, "lsh_weighted.npz")))
