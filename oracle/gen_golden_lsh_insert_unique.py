"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_insert_unique.npz from the REAL reference's streaming dedup loop
(MinHashLSH.query, MinHash.jaccard, MinHashLSH.insert).

Run where an ekzhu/datasketch checkout exists (it imports the reference from it), after oracle/gen_golden.py has
written tests/golden/lsh.npz, whose 300 signatures it indexes:

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_insert_unique.py

The 300 documents of lsh.npz are rebuilt as gen_golden_lsh_query_jaccard.py does.  The batch is held out: perturbed
copies of indexed documents, drift chains (each document a perturbed copy of the one before it), exact copies within the
batch and unrelated documents, shuffled.  For each threshold t (None: any candidate, 0.5, 0.8, 0.9) a fresh
MinHashLSH(0.8, 128) holding the 300 documents runs

    for m in batch:
        if not [d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]:
            lsh.insert(300 + kept_so_far, m)

and the file stores, per row, whether it was kept and, for a dropped row, the candidate with the largest
MinHash.jaccard (the smallest key among equal ones) and that Jaccard value (-1 for kept rows).  It pins the oracle of
tests/test_lsh_insert_unique.py and the CUDA path.
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
from oracle.gen_golden_lsh_query_jaccard import ident, lsh_docs  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
THRESHOLDS = (None, 0.5, 0.8, 0.9)


def _perturb(rs, doc, frac):
    q = doc.copy()
    nres = max(1, int(round(len(q) * frac)))
    q[rs.choice(len(q), nres, replace=False)] = rs.randint(0, 2 ** 32, size=nres, dtype=np.uint64)
    return q


def gen_lsh_insert_unique():
    sig = np.load(os.path.join(OUT, "lsh.npz"))["sig"]
    docs = lsh_docs()
    ms = MinHash.bulk([[int(t) for t in doc] for doc in docs], num_perm=128, seed=1, hashfunc=ident)
    assert np.array_equal(np.stack([m.hashvalues for m in ms]).astype(np.uint32), sig), "lsh.npz was made differently"
    rs = np.random.RandomState(47)
    batch, kinds = [], []
    for j, i in enumerate(rs.choice(300, 40, replace=False).tolist()):   # perturbed copies of indexed documents
        batch.append(_perturb(rs, docs[i], (0.02, 0.05, 0.1, 0.2)[j % 4]))
        kinds.append(1)
    for _ in range(10):                                                  # drift chains of 6: 10 % resampled per step
        cur = rs.randint(0, 2 ** 32, size=rs.randint(40, 80), dtype=np.uint64)
        for _ in range(6):
            batch.append(cur)
            kinds.append(3)
            cur = _perturb(rs, cur, 0.1)
    fresh = [rs.randint(0, 2 ** 32, size=rs.randint(20, 80), dtype=np.uint64) for _ in range(30)]
    batch.extend(fresh)                                                  # unrelated documents
    kinds.extend([0] * len(fresh))
    for i in rs.choice(len(batch), 15, replace=False).tolist():          # exact copies within the batch
        batch.append(batch[i].copy())
        kinds.append(2)
    order = rs.permutation(len(batch))
    chain_pos = [j for j in order.tolist() if kinds[j] == 3]
    # keep each chain in order (a chain's steps are consecutive in `batch`), the rest shuffled around it
    it = iter(sorted(chain_pos))
    order = [next(it) if kinds[j] == 3 else j for j in order.tolist()]
    batch = [batch[j] for j in order]
    kinds = [kinds[j] for j in order]
    bs = MinHash.bulk([[int(t) for t in q] for q in batch], num_perm=128, seed=1, hashfunc=ident)
    d = {"b_r": None, "batch": np.stack([m.hashvalues for m in bs]).astype(np.uint32),
         "kind": np.array(kinds, dtype=np.int8),
         "thresholds": np.array([-1.0 if t is None else t for t in THRESHOLDS], dtype=np.float64)}
    for j, t in enumerate(THRESHOLDS):
        lsh = MinHashLSH(threshold=0.8, num_perm=128)
        held = {}
        for i, m in enumerate(ms):
            lsh.insert(i, m)
            held[i] = m
        d["b_r"] = np.array([lsh.b, lsh.r], dtype=np.int64)
        kept, match, jac = [], [], []
        for m in bs:
            cand = [c for c in lsh.query(m) if t is None or m.jaccard(held[c]) >= t]
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
        d["kept%d" % j] = np.array(kept, dtype=np.int8)
        d["match%d" % j] = np.array(match, dtype=np.int64)
        d["jaccard%d" % j] = np.array(jac, dtype=np.float64)
    np.savez_compressed(os.path.join(OUT, "lsh_insert_unique.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_lsh_insert_unique()
    print("lsh_insert_unique.npz", os.path.getsize(os.path.join(OUT, "lsh_insert_unique.npz")))
