"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_topk.npz from the REAL reference's MinHashLSH.query and
MinHash.jaccard.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it), after oracle/gen_golden.py has
written tests/golden/lsh.npz, whose 300 signatures it indexes:

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_topk.py

The 300 documents of lsh.npz are rebuilt as gen_golden_lsh_query_jaccard.py rebuilds them (and checked against their
signatures).  The queries are held-out documents: perturbed copies of indexed ones, exact copies and unrelated ones; the
indexed documents themselves are asked too, without themselves.  Everything stored is an output of the unmodified
reference's public API (``MinHash.bulk``, ``MinHashLSH.insert`` / ``query``, ``MinHash.jaccard``): per query and per
(k, t), the list ``sorted([d for d in lsh.query(m) if m.jaccard(doc[d]) >= t], key=lambda d: (-m.jaccard(doc[d]),
d))[:k]`` and those Jaccard values, padded with -1 to k entries.  It pins the oracle of tests/test_lsh_topk.py and the
CUDA path.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle.gen_golden_lsh_query_jaccard import OUT, datasketch, ident, lsh_docs  # noqa: E402  (imports the reference)
from datasketch import MinHash, MinHashLSH  # noqa: E402

KS = (1, 5, 32)
THRESHOLDS = (None, 0.5, 0.8)


def topk(lsh, m, ms, k, t, exclude=None):
    cand = [d for d in lsh.query(m) if d != exclude and (t is None or m.jaccard(ms[d]) >= t)]
    best = sorted(cand, key=lambda d: (-m.jaccard(ms[d]), d))[:k]
    idx = np.full(k, -1, dtype=np.int64)
    jac = np.full(k, -1.0, dtype=np.float64)
    idx[:len(best)] = best
    jac[:len(best)] = [m.jaccard(ms[d]) for d in best]
    return idx, jac


def gen_lsh_topk():
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    docs = lsh_docs()
    ms = MinHash.bulk([[int(t) for t in doc] for doc in docs], num_perm=128, seed=1, hashfunc=ident)
    assert np.array_equal(np.stack([m.hashvalues for m in ms]).astype(np.uint32), sig), "lsh.npz was made differently"
    lsh = MinHashLSH(threshold=0.8, num_perm=128)
    for i, m in enumerate(ms):
        lsh.insert(i, m)
    rs = np.random.RandomState(47)
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
         "kind": np.array(kinds, dtype=np.int8), "ks": np.array(KS, dtype=np.int64),
         "thresholds": np.array([-1.0 if t is None else t for t in THRESHOLDS], dtype=np.float64)}
    for kk in KS:
        for j, t in enumerate(THRESHOLDS):
            q = [topk(lsh, m, ms, kk, t) for m in qs]                          # held-out queries
            s = [topk(lsh, m, ms, kk, t, exclude=i) for i, m in enumerate(ms)]   # each indexed document without itself
            d["q_k%d_t%d_idx" % (kk, j)] = np.stack([x[0] for x in q])
            d["q_k%d_t%d_jac" % (kk, j)] = np.stack([x[1] for x in q])
            d["s_k%d_t%d_idx" % (kk, j)] = np.stack([x[0] for x in s])
            d["s_k%d_t%d_jac" % (kk, j)] = np.stack([x[1] for x in s])
    np.savez_compressed(os.path.join(OUT, "lsh_topk.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_lsh_topk()
    print("lsh_topk.npz", os.path.getsize(os.path.join(OUT, "lsh_topk.npz")))
