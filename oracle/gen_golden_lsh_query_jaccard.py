"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_query_jaccard.npz from the REAL reference's MinHashLSH.query and
MinHash.jaccard.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it), after oracle/gen_golden.py has
written tests/golden/lsh.npz, whose 300 signatures it indexes:

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_query_jaccard.py

The 300 documents of lsh.npz are rebuilt from gen_golden.py's seed (and checked against its signatures); the queries are
held-out documents: perturbed copies of indexed ones, exact copies and unrelated ones.  Everything stored is an output
of the unmodified reference's public API (``MinHash.bulk``, ``MinHashLSH.insert`` / ``query``, ``MinHash.jaccard``): per
query, the candidate list, each candidate's Jaccard value and the lists ``[d for d in lsh.query(m) if m.jaccard(doc[d]) >=
t]`` for a few thresholds t.  It pins the oracle of tests/test_lsh_query_jaccard.py and the CUDA path.
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
from datasketch import MinHash, MinHashLSH  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
THRESHOLDS = (0.5, 0.8, 0.9)


def ident(x):
    return int(x)


def lsh_docs():
    """The 300 token lists of gen_golden.gen_lsh (same seed, same draws)."""
    rs = np.random.RandomState(21)
    docs = [rs.randint(0, 2 ** 32, size=rs.randint(20, 80), dtype=np.uint64) for _ in range(300)]
    for i in range(0, 300, 3):
        src = docs[i].copy()
        nres = max(1, len(src) // 12)
        src[rs.choice(len(src), nres, replace=False)] = rs.randint(0, 2 ** 32, size=nres, dtype=np.uint64)
        docs[i + 1] = src
        docs[i + 2] = docs[i].copy()
    return docs


def gen_lsh_query_jaccard():
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    docs = lsh_docs()
    ms = MinHash.bulk([[int(t) for t in doc] for doc in docs], num_perm=128, seed=1, hashfunc=ident)
    assert np.array_equal(np.stack([m.hashvalues for m in ms]).astype(np.uint32), sig), "lsh.npz was made differently"
    lsh = MinHashLSH(threshold=0.8, num_perm=128)
    for i, m in enumerate(ms):
        lsh.insert(i, m)
    rs = np.random.RandomState(43)
    queries, kinds = [], []
    for j, i in enumerate(rs.choice(300, 80, replace=False).tolist()):   # perturbed copies: 2 .. 40 % of tokens resampled
        q = docs[i].copy()
        nres = max(1, int(round(len(q) * (0.02, 0.05, 0.1, 0.2, 0.4)[j % 5])))
        q[rs.choice(len(q), nres, replace=False)] = rs.randint(0, 2 ** 32, size=nres, dtype=np.uint64)
        queries.append(q)
        kinds.append(1)
    for i in rs.choice(300, 10, replace=False).tolist():                 # exact copies of indexed documents
        queries.append(docs[i].copy())
        kinds.append(2)
    for _ in range(30):                                                  # unrelated documents
        queries.append(rs.randint(0, 2 ** 32, size=rs.randint(20, 80), dtype=np.uint64))
        kinds.append(0)
    qs = MinHash.bulk([[int(t) for t in q] for q in queries], num_perm=128, seed=1, hashfunc=ident)
    d = {"b_r": np.array([lsh.b, lsh.r], dtype=np.int64), "qsig": np.stack([m.hashvalues for m in qs]).astype(np.uint32),
         "kind": np.array(kinds, dtype=np.int8), "thresholds": np.array(THRESHOLDS, dtype=np.float64)}
    res, jac, ptr = [], [], [0]
    kept = {t: ([], [0]) for t in THRESHOLDS}
    for m in qs:
        cand = sorted(lsh.query(m))
        res.extend(cand)
        jac.extend(m.jaccard(ms[c]) for c in cand)
        ptr.append(len(res))
        for t in THRESHOLDS:
            lst, p = kept[t]
            lst.extend(sorted(c for c in lsh.query(m) if m.jaccard(ms[c]) >= t))
            p.append(len(lst))
    d["query_ptr"], d["query_idx"] = np.array(ptr, dtype=np.int64), np.array(res, dtype=np.int64)
    d["query_jaccard"] = np.array(jac, dtype=np.float64)
    for j, t in enumerate(THRESHOLDS):
        d["kept%d_ptr" % j] = np.array(kept[t][1], dtype=np.int64)
        d["kept%d_idx" % j] = np.array(kept[t][0], dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "lsh_query_jaccard.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_lsh_query_jaccard()
    print("lsh_query_jaccard.npz", os.path.getsize(os.path.join(OUT, "lsh_query_jaccard.npz")))
