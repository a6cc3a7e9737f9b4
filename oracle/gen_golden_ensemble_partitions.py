"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/ensemble_partitions.npz from the REAL reference's size partitioner
(datasketch/lshensemble_partition.py).

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_ensemble_partitions.py

Distributions of distinct set sizes (ascending ``sizes``, ``counts`` > 0), in three families:

* ``heavy``: D in {1, 2, 7, 8, 9, 64, 128, 129, 136, 257, 400} distinct sizes spread log-uniformly up to 10^9, with
  Pareto (heavy-tailed) counts up to about 10^6;
* ``ties``: power-of-two sizes 1, 2, 4, ... with counts in 1..4, so that every term and every sum of the cost table is
  exact and equal totals (ties in the argmins) are common;
* ``sweep``: 80 seeded small distributions (D < 40, sizes up to 60, counts up to 5), each with one num_part < 12; the
  reference's back-tracking reads the p-interval table where its recurrence used the (p-1)-interval one, and in most of
  these cases that changes the bounds (``quirk`` flags them).

Distribution d: ``sizes[dist_ptr[d]:dist_ptr[d+1]]`` and ``counts[...]`` (int64), and ``cost_sha256[d]``: the SHA-256 of
the upper triangle of the reference's ``_compute_nfps_real(counts, sizes)`` as little-endian float64 bit patterns,
column-major (entry (l, u) at u(u+1)/2 + l); for the heavy and tie families up to D = 64 also ``d{d}_cost``, the triangle
itself as uint64 (the digest keeps the file small: a triangle of D = 400 is 640 KB of incompressible bits).
Case c: ``cases[c] = (d, num_part, quirk)``, and ``lowers`` / ``uppers[case_ptr[c]:case_ptr[c+1]]`` (int64), the reference's
``optimal_partitions(sizes, counts, num_part)``.
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
from datasketch.lshensemble_partition import _compute_nfps_real, optimal_partitions  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
HEAVY_D = [1, 2, 7, 8, 9, 64, 128, 129, 136, 257, 400]
TIES_D = [1, 2, 7, 8, 9, 16, 40]


def heavy(rs, d):
    sizes = np.unique(np.exp(rs.uniform(0, np.log(1e9), 4 * d + 8)).astype(np.int64) + 1)
    while len(sizes) < d:
        sizes = np.unique(np.append(sizes, rs.randint(1, 10 ** 9, d)))
    sizes = np.sort(rs.choice(sizes, d, replace=False))
    sizes[-1] = 10 ** 9 if d > 1 else sizes[-1]
    sizes = np.unique(sizes)
    counts = np.minimum((rs.pareto(0.8, len(sizes)) * 3 + 1).astype(np.int64), 10 ** 6)
    return sizes.astype(np.int64), counts


def ties(rs, d):
    return (2 ** np.arange(d, dtype=np.int64)), rs.randint(1, 5, d).astype(np.int64)


def sweep(rs):
    d = int(rs.randint(4, 40))
    sizes = np.sort(rs.choice(np.arange(1, 61), d, replace=False)).astype(np.int64)
    return sizes, rs.randint(1, 6, d).astype(np.int64), int(rs.randint(3, min(12, d)))


def bounds_without_quirk(sizes, nfps, num_part):
    """The same dynamic programme with the back-tracking reading the table its recurrence filled (p-1 intervals)."""
    n = len(sizes)
    last = n - 1
    tab = {1: nfps[0]}
    for p in range(2, num_part):
        t = np.zeros(n)
        for u in range(p - 1, n):
            t[u] = min(tab[p - 1][u1] + nfps[u1 + 1, u] for u1 in range(p - 2, u))
        tab[p] = t
    u = last
    uppers = [last]
    for p in range(num_part, 1, -1):
        u = min((tab[p - 1][u1] + nfps[u1 + 1, u], u1) for u1 in range(p - 2, u))[1]
        uppers.insert(0, u)
    return [int(sizes[x]) for x in uppers]


def triangle_bits(nfps):
    n = nfps.shape[0]
    return np.concatenate([nfps[:u + 1, u] for u in range(n)]).view(np.uint64) if n else np.zeros(0, np.uint64)


def gen():
    rs = np.random.RandomState(20261017)
    d = {}
    dists, cases = [], []
    for dd in HEAVY_D:
        s, c = heavy(rs, dd)
        dists.append((s, c, [1, 2, 3, 8, 16, 32, dd - 1, dd, dd + 1]))
    for dd in TIES_D:
        s, c = ties(rs, dd)
        dists.append((s, c, [1, 2, 3, 8, 16, 32, dd - 1, dd, dd + 1]))
    for _ in range(80):
        s, c, k = sweep(rs)
        dists.append((s, c, [k]))
    n_quirk = 0
    digests, lowers, all_uppers, case_ptr = [], [], [], [0]
    for i, (sizes, counts, parts) in enumerate(dists):
        nfps = _compute_nfps_real(counts, sizes)
        bits = triangle_bits(nfps)
        digests.append(hashlib.sha256(bits.astype("<u8").tobytes()).hexdigest())
        if len(parts) > 1 and len(sizes) <= 64:
            d["d%d_cost" % i] = bits
        for k in sorted({k for k in parts if k >= 1}):
            b = optimal_partitions(sizes, counts, k)
            uppers = [int(x[1]) for x in b]
            quirk = 2 < k < len(sizes) and bounds_without_quirk(sizes, nfps, k) != uppers
            n_quirk += quirk
            c = len(cases)
            cases.append((i, k, int(quirk)))
            lowers.extend(int(x[0]) for x in b)
            all_uppers.extend(uppers)
            case_ptr.append(len(all_uppers))
    d["cases"] = np.array(cases, dtype=np.int64)
    d["case_ptr"] = np.array(case_ptr, dtype=np.int64)
    d["lowers"], d["uppers"] = np.array(lowers, dtype=np.int64), np.array(all_uppers, dtype=np.int64)
    d["dist_ptr"] = np.cumsum([0] + [len(x[0]) for x in dists]).astype(np.int64)
    d["sizes"] = np.concatenate([x[0] for x in dists]).astype(np.int64)
    d["counts"] = np.concatenate([x[1] for x in dists]).astype(np.int64)
    d["cost_sha256"] = np.array(digests)
    np.savez_compressed(os.path.join(OUT, "ensemble_partitions.npz"), **d)
    print("distributions", len(dists), "cases", len(cases), "back-tracking quirk changes the bounds in", n_quirk)


if __name__ == "__main__":
    print("reference:", datasketch.__file__)
    gen()
    print("ensemble_partitions.npz", os.path.getsize(os.path.join(OUT, "ensemble_partitions.npz")))
