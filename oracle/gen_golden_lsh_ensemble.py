"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/lsh_ensemble.npz from the REAL reference's MinHashLSHEnsemble.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_lsh_ensemble.py

Three corpora of sets drawn from one vocabulary, with heavy-tailed sizes and planted subsets and supersets, and held-out
query sets: subsets of indexed sets (down to one token, so upper / size rises above xqs[-1]), supersets (up to thousands
of tokens, so it falls below xqs[0]) and unrelated sets.  Signatures are the reference's ``MinHash.bulk`` of the token ids
(hashfunc = identity, seed 1); the file stores the token ids (they compress, the signatures do not) with the SHA-256 of
each signature matrix, so a test can rebuild the matrices and check them.  Per configuration it stores what the
unmodified reference's public API and its own ``_get_optimal_param`` give: ``params``, ``xqs``, ``lowers`` / ``uppers``
(-1 for None), the (b, r) of every (query, partition) (0 where the partition is skipped) and ``sorted(set(query(m,
size)))`` of every query as CSR over row numbers.
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

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
VOCAB = 6000

# name -> (K, number of sets, number of queries, size draw, seed)
CORPORA = {
    "a": (128, 160, 50, "pareto", 7),
    "b": (64, 80, 30, "few", 8),      # few distinct sizes: more partitions than sizes
    "c": (16, 100, 40, "pareto", 9),
}
# (threshold, num_perm, num_part, m, corpus)
CONFIGS = [(0.5, 128, 16, 8, "a"), (0.8, 128, 1, 8, "a"), (0.7, 64, 40, 4, "b"), (0.5, 16, 4, 2, "c")]


def ident(x):
    return int(x)


def draw_sizes(rs, n, how):
    if how == "few":
        return rs.choice([4, 9, 17, 33, 65, 130], size=n)
    return np.clip((rs.pareto(1.1, n) * 6 + 2).astype(np.int64), 2, 900)


def corpus(k, n, nq, how, seed):
    rs = np.random.RandomState(seed)
    sizes = draw_sizes(rs, n, how)
    sets = [rs.choice(VOCAB, int(s), replace=False) for s in sizes]
    for j in rs.choice(n, n // 5, replace=False).tolist():        # planted subsets of other indexed sets
        i = int(rs.randint(n))
        if len(sets[i]) > 2:
            sets[j] = rs.choice(sets[i], int(rs.randint(1, len(sets[i]))), replace=False)
    for j in rs.choice(n, n // 8, replace=False).tolist():        # planted supersets
        i = int(rs.randint(n))
        extra = rs.choice(VOCAB, int(rs.randint(1, 3 * len(sets[i]) + 2)), replace=False)
        sets[j] = np.union1d(sets[i], extra)
    queries = []
    for _ in range(2 * nq // 5):                                  # subsets, down to one token
        src = sets[int(rs.randint(n))]
        queries.append(rs.choice(src, int(rs.randint(1, len(src) + 1)), replace=False))
    for _ in range(nq // 3):                                      # supersets, up to thousands of tokens
        src = sets[int(rs.randint(n))]
        queries.append(np.union1d(src, rs.choice(VOCAB, int(rs.choice([5, 60, 700])), replace=False)))
    queries.append(np.union1d(sets[0], rs.choice(VOCAB, 2000, replace=False)))
    while len(queries) < nq:                                      # unrelated sets
        queries.append(rs.choice(VOCAB, int(draw_sizes(rs, 1, how)[0]), replace=False))
    return sets, queries


def csr(lists, dtype):
    ptr = np.zeros(len(lists) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(x) for x in lists])
    flat = np.concatenate([np.asarray(x, dtype=dtype) for x in lists]) if ptr[-1] else np.zeros(0, dtype=dtype)
    return ptr, flat


def signatures(sets, k):
    ms = MinHash.bulk([[int(t) for t in s] for s in sets], num_perm=k, seed=1, hashfunc=ident)
    sig = np.stack([m.hashvalues for m in ms])
    assert sig.max() < 2 ** 32
    return ms, sig.astype(np.uint32)


def sha(sig):
    return hashlib.sha256(np.ascontiguousarray(sig, dtype="<u4").tobytes()).hexdigest()


def gen():
    d = {}
    built = {}
    for name, (k, n, nq, how, seed) in CORPORA.items():
        sets, queries = corpus(k, n, nq, how, seed)
        ms, sig = signatures(sets, k)
        qms, qsig = signatures(queries, k)
        built[name] = (ms, qms, [len(s) for s in sets], [len(q) for q in queries])
        d[name + "_tok_ptr"], d[name + "_tok"] = csr(sets, np.uint16)
        d[name + "_qtok_ptr"], d[name + "_qtok"] = csr(queries, np.uint16)
        d[name + "_sig_sha256"], d[name + "_qsig_sha256"] = np.array(sha(sig)), np.array(sha(qsig))
    d["configs"] = np.array([c[:4] for c in CONFIGS], dtype=np.float64)
    d["config_corpus"] = np.array([c[4] for c in CONFIGS])
    for c, (thr, k, num_part, m, name) in enumerate(CONFIGS):
        ms, qms, sizes, qsizes = built[name]
        ens = MinHashLSHEnsemble(threshold=thr, num_perm=k, num_part=num_part, m=m)
        ens.index([(i, ms[i], sizes[i]) for i in range(len(ms))])
        d["c%d_params" % c] = np.asarray(ens.params, dtype=np.int64)
        d["c%d_xqs" % c] = np.asarray(ens.xqs, dtype=np.float64)
        d["c%d_lowers" % c] = np.array([-1 if x is None else int(x) for x in ens.lowers], dtype=np.int64)
        d["c%d_uppers" % c] = np.array([-1 if x is None else int(x) for x in ens.uppers], dtype=np.int64)
        bsel = np.zeros((len(qms), num_part), dtype=np.int32)
        rsel = np.zeros((len(qms), num_part), dtype=np.int32)
        res = []
        for q, (mq, size) in enumerate(zip(qms, qsizes)):
            for p, u in enumerate(ens.uppers):
                if u is not None:
                    bsel[q, p], rsel[q, p] = ens._get_optimal_param(u, size)
            res.append(sorted(set(ens.query(mq, size))))
        d["c%d_b" % c], d["c%d_r" % c] = bsel, rsel
        d["c%d_res_ptr" % c], d["c%d_res_idx" % c] = csr(res, np.int32)
        print("config", c, (thr, k, num_part, m), "uppers", d["c%d_uppers" % c].tolist(), "results", len(d["c%d_res_idx" % c]),
              "empty", sum(len(x) == 0 for x in res))
    np.savez_compressed(os.path.join(OUT, "lsh_ensemble.npz"), **d)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen()
    print("lsh_ensemble.npz", os.path.getsize(os.path.join(OUT, "lsh_ensemble.npz")))
