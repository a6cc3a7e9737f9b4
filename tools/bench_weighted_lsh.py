"""GpuLSH(weighted=True) (weighted MinHash signatures in the device index) against the host MinHashLSH.

    python tools/bench_weighted_lsh.py [--vectors 1000000] [--queries 100000] [--host-vectors 20000]
                                       [--host-queries 2000] [--out profiles/h100_weighted_lsh.jsonl]

Corpus (seeded, built on the device): --vectors integer-frequency vectors of dim 512 (weights 1..19, about 60 % zeros);
10 % of them are near-duplicates of others (each non-zero weight dropped with probability 0.1).  Queries: --queries fresh
vectors, half near-duplicates of indexed ones, half unrelated.  Sample size 128, LSH threshold 0.8.
Device: CUDA events around each whole call, after a warm-up of every call on a small index, 3 rounds where the call does not
change the index: WeightedMinHashGenerator.minhash_batch(to_host=False), insert, query_jaccard(0.8) and query_best(0.8) of
the queries, candidate_pairs(0.8), duplicate_clusters() with and without 0.8, and insert_unique(0.8) of the queries (once,
last).
Host: this package's MinHashLSH with WeightedMinHash objects (the reference's dict path) inserts the first --host-vectors
signatures and answers --host-queries queries (near-duplicates of those vectors); a device index over the same signatures
answers the same queries, and the candidate sets and WeightedMinHash.jaccard values are compared.
Prints one JSON line and appends it to --out, with the card's name and power limit read in the same process.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import datasketch_b200 as dsk  # noqa: E402
from datasketch_b200.lsh import MinHashLSH  # noqa: E402
from datasketch_b200.weighted_minhash import WeightedMinHash  # noqa: E402

DIM, SS, THR = 512, 128, 0.8


def gpu_card():
    """The card's name, power limit and top SM clock, read in the same process as the timings beside them."""
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def vectors(n, g):
    x = torch.randint(1, 20, (n, DIM), device="cuda", generator=g).float()
    x *= torch.rand((n, DIM), device="cuda", generator=g) >= 0.6
    x[x.sum(1) == 0, 0] = 1.0
    return x


def near(x, g):
    y = x * (torch.rand(x.shape, device="cuda", generator=g) >= 0.1)
    y[y.sum(1) == 0, 0] = 1.0
    return y


def corpus(n, nq, host_n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = vectors(n, g)
    dup = n // 10
    dst = torch.randperm(n, device="cuda", generator=g)[:dup]
    src = torch.randint(0, n, (dup,), device="cuda", generator=g)
    X[dst] = near(X[src], g)
    Q = vectors(nq, g)
    Q[:nq // 2] = near(X[torch.randint(0, n, (nq // 2,), device="cuda", generator=g)], g)
    HQ = near(X[torch.randint(0, host_n, (nq,), device="cuda", generator=g)], g)   # host queries: near the host's vectors
    return X, Q, HQ


def timed(fn, rounds):
    """(result of the last round, per-round ms) with CUDA events around each whole call."""
    ms, out = [], None
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, [round(x, 3) for x in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vectors", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--host-vectors", type=int, default=20_000)
    ap.add_argument("--host-queries", type=int, default=2_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_weighted_lsh.jsonl"))
    a = ap.parse_args()
    n, nq = a.vectors, a.queries
    rec = {"bench": "weighted_lsh", "command": " ".join(["python"] + sys.argv), "vectors": n, "queries": nq, "dim": DIM,
           "sample_size": SS, "threshold": THR}
    rec.update(gpu_card())
    X, Q, HQ = corpus(n, nq, a.host_vectors)
    rec["zero_share"] = round(float((X == 0).float().mean()), 4)
    mg = dsk.WeightedMinHashGenerator(DIM, sample_size=SS, seed=1)

    # warm-up of every call on a small index
    w = mg.minhash_batch(X[:2000], to_host=False)
    wi = dsk.GpuLSH(threshold=THR, num_perm=SS, capacity=4000, weighted=True)
    wi.insert(w[:1000])
    wi.query_jaccard(w[1000:], THR)
    wi.query_best(w[1000:], THR)
    wi.candidate_pairs(THR)
    wi.duplicate_clusters()
    wi.duplicate_clusters(THR)
    wi.insert_unique(w[1000:], THR)
    del wi, w

    sig, rec["minhash_batch_ms"] = timed(lambda: mg.minhash_batch(X, to_host=False), 3)
    qsig = mg.minhash_batch(Q, to_host=False)
    ix = None

    def build():
        nonlocal ix
        ix = dsk.GpuLSH(threshold=THR, num_perm=SS, capacity=n + nq, weighted=True)
        torch.cuda.synchronize()
        return ix

    rec["b_r"] = [build().b, ix.r]
    _, rec["insert_ms"] = timed(lambda: ix.insert(sig), 1)
    qj, rec["query_jaccard_ms"] = timed(lambda: ix.query_jaccard(qsig, THR, to_host=False), 3)
    rec["query_jaccard_kept"] = int(qj[0][-1])
    qb, rec["query_best_ms"] = timed(lambda: ix.query_best(qsig, THR, to_host=False), 3)
    rec["query_best_hits"] = int((qb[0] >= 0).sum())
    cp, rec["candidate_pairs_ms"] = timed(lambda: ix.candidate_pairs(THR, to_host=False), 3)
    rec["candidate_pairs"] = int(cp[0][-1])
    lab, rec["duplicate_clusters_ms"] = timed(lambda: ix.duplicate_clusters(to_host=False), 3)
    rec["clusters"] = int((lab == torch.arange(n, device=lab.device, dtype=lab.dtype)).sum())
    lab, rec["duplicate_clusters_filtered_ms"] = timed(lambda: ix.duplicate_clusters(THR, to_host=False), 3)
    rec["clusters_filtered"] = int((lab == torch.arange(n, device=lab.device, dtype=lab.dtype)).sum())
    ku, rec["insert_unique_ms"] = timed(lambda: ix.insert_unique(qsig, THR, to_host=False), 1)
    rec["insert_unique_kept"] = int(ku[0].sum())
    del ix, sig, qsig, qj, qb, cp, lab, ku
    torch.cuda.empty_cache()

    # host MinHashLSH over WeightedMinHash objects, and the device on the same signatures
    hn, hq = a.host_vectors, a.host_queries
    hsig = mg.minhash_batch(X[:hn], to_host=False)
    hqsig = mg.minhash_batch(HQ[:hq], to_host=False)
    hs, hqs = hsig.cpu().numpy(), hqsig.cpu().numpy()
    ms = [WeightedMinHash(1, hs[i]) for i in range(hn)]
    qs = [WeightedMinHash(1, hqs[i]) for i in range(hq)]
    host = MinHashLSH(threshold=THR, num_perm=SS)
    t0 = time.perf_counter()
    for i, m in enumerate(ms):
        host.insert(i, m)
    rec["host_insert_us_per_vector"] = round((time.perf_counter() - t0) / hn * 1e6, 2)
    t0 = time.perf_counter()
    hres = [host.query(m) for m in qs]
    rec["host_query_us_per_query"] = round((time.perf_counter() - t0) / hq * 1e6, 2)
    dix = dsk.GpuLSH(threshold=THR, num_perm=SS, capacity=hn, weighted=True)
    dix.insert(hsig)
    ptr, idx, eq = dix.query_jaccard(hqsig)
    same = True
    for q in range(hq):
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        got = dict(zip(idx[sl].tolist(), eq[sl].tolist()))
        same = same and set(got) == set(hres[q]) and all(
            got[d] / float(SS) == qs[q].jaccard(ms[d]) for d in hres[q])
    rec["host_candidates"] = int(sum(len(x) for x in hres))
    rec["device_equals_host"] = bool(same)
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
