"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_ensemble_containment.npz from the REAL reference's
MinHashLSHEnsemble and MinHash.jaccard.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_ensemble_containment.py

The corpora are those of tests/golden/lsh_ensemble.npz, rebuilt from the token ids stored there; their signatures are
the reference's ``MinHash.bulk`` (hashfunc = identity, seed 1) at each configuration's K, stored as SHA-256 digests so a
test can rebuild and check them.  The configurations add what that fixture lacks: K = 100, K = 320 with m = 2, and sizes
that are the true sizes times 10^13 plus a seeded offset (s_q + s_x above 2^53, where int -> float rounding matters).
For every query (m, s) it stores each candidate x of ``ens.query(m, s)`` with its eq and the float64 bits of

    c = m.jaccard(m_x) * (s + s_x) / (s * (1 + m.jaccard(m_x)))      (Python ints and floats, evaluated as written)

and for every indexed set i the same for ``ens.query(ms[i], sizes[i])`` without i.  Thresholds and top-k cuts are
applied by the tests from these bits.  Running it twice gives equal arrays (the .npz container itself carries times).
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

REF = os.environ["DATASKETCH_REF"]
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import fake_backends  # noqa: E402  in-memory stand-ins for the optional `redis` / `pybloomfilter` packages
fake_backends.install()           # must precede the import below: storage.py / lsh_bloom.py probe them at import time
import datasketch  # noqa: E402  (the reference)
from datasketch import MinHash, MinHashLSHEnsemble  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden")
BIG = 10 ** 13

# (threshold, num_perm, num_part, m, corpus of lsh_ensemble.npz, big sizes)
CONFIGS = [
    (0.5, 128, 16, 8, "a", 0),    # the default-like configuration
    (0.7, 64, 40, 4, "b", 0),     # more partitions than sizes: trailing None upper bounds
    (0.5, 100, 8, 4, "a", 0),     # K = 100: the integer form of the estimate rounds differently here
    (0.4, 320, 4, 2, "c", 0),     # K = 320, small m
    (0.5, 128, 16, 8, "a", 1),    # sizes * 10^13 + offset: s_q + s_x above 2^53
    (0.6, 100, 6, 4, "c", 1),
]


def ident(x):
    return int(x)


def sets_of(g, name, which):
    ptr, tok = g[name + "_" + which + "tok_ptr"], g[name + "_" + which + "tok"]
    return [tok[ptr[i]:ptr[i + 1]].astype(np.int64).tolist() for i in range(len(ptr) - 1)]


def big_sizes(sizes, seed):
    rs = np.random.RandomState(seed)
    return [int(s) * BIG + int(o) for s, o in zip(sizes, rs.randint(0, BIG // 10, size=len(sizes)))]


def containment(mq, mx, sq, sx):
    j = mq.jaccard(mx)
    return j * (sq + sx) / (sq * (1 + j))


def csr_of(rows):
    """rows: per query a sorted list of (x, eq, c) -> ptr, idx, eq, c bits (uint64)."""
    ptr = np.zeros(len(rows) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(r) for r in rows])
    flat = [t for r in rows for t in r]
    idx = np.array([t[0] for t in flat], dtype=np.int32)
    eq = np.array([t[1] for t in flat], dtype=np.int32)
    cb = np.array([t[2] for t in flat], dtype=np.float64).view(np.uint64)
    return ptr, idx, eq, cb


def sha(sig):
    return hashlib.sha256(np.ascontiguousarray(sig, dtype="<u4").tobytes()).hexdigest()


def gen():
    g = np.load(os.path.join(OUT, "lsh_ensemble.npz"))
    d = {"configs": np.array([c[:4] for c in CONFIGS], dtype=np.float64),
         "config_corpus": np.array([c[4] for c in CONFIGS]),
         "config_big": np.array([c[5] for c in CONFIGS], dtype=np.int64)}
    for c, (thr, k, num_part, m, name, big) in enumerate(CONFIGS):
        sets, queries = sets_of(g, name, ""), sets_of(g, name, "q")
        ms = MinHash.bulk(sets, num_perm=k, seed=1, hashfunc=ident)
        qms = MinHash.bulk(queries, num_perm=k, seed=1, hashfunc=ident)
        d["c%d_sig_sha256" % c] = np.array(sha(np.stack([x.hashvalues for x in ms]).astype(np.uint32)))
        d["c%d_qsig_sha256" % c] = np.array(sha(np.stack([x.hashvalues for x in qms]).astype(np.uint32)))
        sizes, qsizes = [len(s) for s in sets], [len(q) for q in queries]
        if big:
            sizes, qsizes = big_sizes(sizes, 100 + c), big_sizes(qsizes, 200 + c)
        d["c%d_sizes" % c], d["c%d_qsizes" % c] = np.array(sizes, dtype=np.int64), np.array(qsizes, dtype=np.int64)
        ens = MinHashLSHEnsemble(threshold=thr, num_perm=k, num_part=num_part, m=m)
        ens.index([(i, ms[i], sizes[i]) for i in range(len(ms))])
        d["c%d_uppers" % c] = np.array([-1 if x is None else int(x) for x in ens.uppers], dtype=np.int64)

        def rows(mq, sq, skip):
            xs = sorted(set(ens.query(mq, sq)) - {skip})
            return [(x, int(np.count_nonzero(mq.hashvalues == ms[x].hashvalues)), containment(mq, ms[x], sq, sizes[x]))
                    for x in xs]
        q_rows = [rows(mq, sq, None) for mq, sq in zip(qms, qsizes)]
        s_rows = [rows(ms[i], sizes[i], i) for i in range(len(ms))]
        for key, rr in (("q", q_rows), ("s", s_rows)):
            d["c%d_%s_ptr" % (c, key)], d["c%d_%s_idx" % (c, key)], d["c%d_%s_eq" % (c, key)], d["c%d_%s_cbits" % (c, key)] = \
                csr_of(rr)
        allc = [t[2] for r in q_rows + s_rows for t in r]
        print("config", c, (thr, k, num_part, m, name, big), "query candidates", sum(len(r) for r in q_rows),
              "self candidates", sum(len(r) for r in s_rows), "c > 1:", sum(x > 1 for x in allc),
              "max s_q + s_x > 2^53:", max(sizes) + max(qsizes) > 2 ** 53)
    np.savez_compressed(os.path.join(OUT, "lsh_ensemble_containment.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen()
    print("lsh_ensemble_containment.npz", os.path.getsize(os.path.join(OUT, "lsh_ensemble_containment.npz")))
