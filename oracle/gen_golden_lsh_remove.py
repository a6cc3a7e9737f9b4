"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_remove.npz from the REAL reference's MinHashLSH.remove.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it), after oracle/gen_golden.py has
written tests/golden/lsh.npz, whose 300 signatures it indexes:

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_remove.py

The query lists it stores are outputs of the unmodified reference's public API (``MinHash``, ``MinHashLSH.insert`` /
``remove`` / ``query``); they pin the removal oracle of tests/test_lsh_remove.py and the CUDA path.
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


def gen_lsh_remove():
    """MinHashLSH.remove over lsh.npz's 300 signatures (keys 0..299; docs 3j, 3j+1, 3j+2 are an original, a
    near-duplicate and an exact duplicate): query of every row after removals, and again after some keys came back."""
    g = np.load(os.path.join(OUT, "lsh.npz"))
    sig = g["sig"]
    ms = [MinHash(num_perm=128, hashvalues=row.astype(np.uint64)) for row in sig]
    lsh = MinHashLSH(threshold=0.8, num_perm=128)
    for i, m in enumerate(ms):
        lsh.insert(i, m)
    removed = [2, 5,                 # exact duplicates: the last-inserted member of their buckets
               4, 7,                 # near-duplicates
               9, 10, 11, 60, 61, 62,  # whole triples: every bucket only they share becomes empty
               12, 24, 36,           # originals: the first-inserted member of their buckets
               16, 28,               # the middle member
               150, 151, 299]
    for key in removed:
        lsh.remove(key)

    def queries():
        res, ptr = [], [0]
        for m in ms:
            res.extend(sorted(lsh.query(m)))
            ptr.append(len(res))
        return np.array(ptr, dtype=np.int64), np.array(res, dtype=np.int64)

    d = {"removed": np.array(removed, dtype=np.int64), "b_r": np.array([lsh.b, lsh.r], dtype=np.int64)}
    d["query_ptr"], d["query_idx"] = queries()
    reinserted = [2, 10, 24, 299]
    for key in reinserted:
        lsh.insert(key, ms[key])
    d["reinserted"] = np.array(reinserted, dtype=np.int64)
    d["query2_ptr"], d["query2_idx"] = queries()
    np.savez_compressed(os.path.join(OUT, "lsh_remove.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen_lsh_remove()
    print("lsh_remove.npz", os.path.getsize(os.path.join(OUT, "lsh_remove.npz")))
