"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/wmh_sparse.npz from the REAL reference's WeightedMinHashGenerator on a
scipy.sparse.csr_matrix at a large dimension (its own sparse entry point, minhash_many, weighted_minhash.py:161-247) and
its minhash on some of those rows densified.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_wmh_sparse.py

dim 200,003, sample_size 128, seed 7; 320 rows with Zipf(1.1)-distributed columns and 0 to 3,000 stored entries each:
all-zero rows, rows of one and two entries, integer counts, tiny weights (negative logarithms) and lognormal weights.
The matrix is stored as CSR arrays (float32 data, no explicit zeros: the reference's nonzero() would skip them).  The
generator's parameters (3 x 98 MB) are not stored: the tests regenerate them with oracle_np.wmh_params and check them
against the float64 sums kept here.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

REF = os.environ["DATASKETCH_REF"]
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import fake_backends  # noqa: E402  in-memory stand-ins for the optional `redis` / `pybloomfilter` packages
fake_backends.install()           # must precede the import below: storage.py / lsh_bloom.py probe them at import time
import scipy.sparse  # noqa: E402
from datasketch import WeightedMinHashGenerator  # noqa: E402  (the reference)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
DIM, SS, SEED, N, N_DENSE = 200_003, 128, 7, 320, 24


def _matrix(rs):
    lens = np.minimum(rs.zipf(1.6, N) * 20, 3000)
    lens[:6] = [0, 1, 2, 0, 3000, 2999]
    lens[rs.choice(np.arange(6, N), 10, replace=False)] = 0
    lens[-1] = 0
    rows, cols, vals = [], [], []
    for i, ln in enumerate(lens):
        c = np.unique((rs.zipf(1.1, 4 * ln + 8) - 1) % DIM)
        c = np.sort(rs.permutation(c)[:ln])
        kind = i % 4
        if kind == 0 or kind == 1:
            v = rs.randint(1, 30, len(c)).astype(np.float32)            # integer counts
        elif kind == 2:
            v = rs.uniform(1e-6, 1e-3, len(c)).astype(np.float32)       # tiny weights: negative logs
        else:
            v = rs.lognormal(0, 2, len(c)).astype(np.float32)
        rows.append(np.full(len(c), i))
        cols.append(c)
        vals.append(v)
    X = scipy.sparse.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(N, DIM),
                                dtype=np.float32)
    assert X.has_canonical_format and (X.data > 0).all()
    return X


def main():
    rs = np.random.RandomState(2024)
    X = _matrix(rs)
    g = WeightedMinHashGenerator(DIM, SS, SEED)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        many = g.minhash_many(X)
    null = np.array([m is None for m in many])
    assert (null == (np.diff(X.indptr) == 0)).all()
    many_out = np.zeros((N, SS, 2), dtype=np.int64)
    for i, m in enumerate(many):
        if m is not None:
            many_out[i] = m.hashvalues
    nonempty = np.where(~null)[0]
    dense_rows = np.unique(np.concatenate([nonempty[:4], rs.choice(nonempty, N_DENSE - 4, replace=False)]))
    dense_rows = dense_rows[:N_DENSE]
    dense_out = np.stack([g.minhash(X[i].toarray().ravel()).hashvalues for i in dense_rows]).astype(np.int64)
    d = dict(cfg=np.array([DIM, SS, SEED], dtype=np.int64),
             indptr=X.indptr.astype(np.int64), indices=X.indices.astype(np.int32), data=X.data,
             many_out=many_out, many_null=null, dense_rows=dense_rows.astype(np.int64), dense_out=dense_out,
             param_sums=np.array([g.rs.astype(np.float64).sum(), g.ln_cs.astype(np.float64).sum(),
                                  g.betas.astype(np.float64).sum()]))
    np.savez_compressed(os.path.join(OUT, "wmh_sparse.npz"), **d)
    print("wrote wmh_sparse.npz: %d rows, %d entries, %d empty" % (N, X.nnz, int(null.sum())))


if __name__ == "__main__":
    main()
