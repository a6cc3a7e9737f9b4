"""GpuLSHForest: index(), query, the ranked query_topk / neighbors and the flows they replace, against the host class.

    python tools/bench_forest.py [--docs 1000000] [--queries 100000] [--host-docs 20000] [--rounds 3]
                                 [--out profiles/h100_forest.jsonl]

Corpus (seeded): --docs random 128-value MinHash rows with planted near-duplicates (copies of other rows with 5 / 15 / 30 %
of the positions re-drawn); queries are indexed rows with 10 % of the positions re-drawn.  The weighted forest indexes
--docs weighted signatures (sample size 128) of dim-256 integer-frequency vectors from WeightedMinHashGenerator.
Device: CUDA events around each whole call, after a warm-up of every call, --rounds rounds (min and max reported):
index() unweighted and weighted, query(sig, 10), query_topk(10) and query_topk(10, candidates=100) beside the flow they
replace (query + codec.jaccard_pairs + a torch sort, outputs checked equal first), neighbors(10).
Host: MinHashLSHForest over --host-docs of the rows, and the reference docstring's post-processing (query(m, 2k), a
jaccard per key, keep the best k) for 2,000 queries, per query; its lists are checked against query_topk first.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import datasketch_b200 as dsk  # noqa: E402
from test_lshforest_topk import _planted, flow_topk  # noqa: E402

K, L = 128, 8


def gpu_card():
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def timed(fn, rounds):
    fn()                                                  # warm-up
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return [round(min(out), 3), round(max(out), 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--host-docs", type=int, default=20_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_forest.jsonl"))
    a = ap.parse_args()
    rs = np.random.RandomState(0)
    res = {"card": gpu_card(), "cmd": " ".join(sys.argv), "docs": a.docs, "queries": a.queries, "K": K, "l": L}
    sig = _planted(rs, a.docs, K, a.docs // 10)
    q = sig[rs.randint(0, a.docs, a.queries)].copy()
    flip = rs.rand(*q.shape) < 0.1
    q[flip] = rs.randint(0, 1 << 32, size=int(flip.sum()), dtype=np.uint64).astype(np.uint32)
    d_sig, d_q = torch.from_numpy(sig.view(np.int32)).cuda(), torch.from_numpy(q.view(np.int32)).cuda()
    dev = dsk.GpuLSHForest(num_perm=K, l=L)
    dev.add(d_sig)
    res["index_ms"] = timed(dev.index, a.rounds)

    mg = dsk.WeightedMinHashGenerator(256, 128, seed=1)
    g = torch.Generator(device="cuda").manual_seed(1)
    X = torch.randint(1, 20, (a.docs, 256), device="cuda", generator=g).float()
    X *= torch.rand(X.shape, device="cuda", generator=g) >= 0.6
    X[:, 0] += 1
    wdev = dsk.GpuLSHForest(num_perm=128, l=L, weighted=True)
    for s in range(0, a.docs, 250_000):
        wdev.add(mg.minhash_batch(X[s:s + 250_000], to_host=False))
    del X
    res["index_weighted_ms"] = timed(wdev.index, a.rounds)
    del wdev

    res["query10_ms"] = timed(lambda: dev.query(d_q, 10, to_host=False), a.rounds)
    for k, c, tag in ((10, 20, "topk10"), (10, 100, "topk10_c100")):
        idx, eq = dev.query_topk(d_q, k, candidates=c, to_host=False)
        w_idx, w_eq = flow_topk(dsk, dev, d_q, k, c)
        res[tag + "_equal"] = bool(torch.equal(idx, w_idx) and torch.equal(eq, w_eq))
        res[tag + "_ms"] = timed(lambda: dev.query_topk(d_q, k, candidates=c, to_host=False), a.rounds)
        res[tag + "_flow_ms"] = timed(lambda: flow_topk(dsk, dev, d_q, k, c), a.rounds)
    res["neighbors10_ms"] = timed(lambda: dev.neighbors(10, to_host=False), a.rounds)

    # host: MinHashLSHForest + the post-processing loop of the reference's query docstring
    hn = a.host_docs
    hsig = sig[:hn]
    host = dsk.MinHashLSHForest(num_perm=K, l=L)
    ms = [dsk.LeanMinHash(seed=1, hashvalues=r.astype(np.uint64)) for r in hsig]
    t0 = time.perf_counter()
    for i, m in enumerate(ms):
        host.add(i, m)
    host.index()
    res["host_index_s"] = round(time.perf_counter() - t0, 3)
    small = dsk.GpuLSHForest(num_perm=K, l=L)
    small.add(hsig)
    small.index()
    qs = q[:2000]
    qm = [dsk.LeanMinHash(seed=1, hashvalues=r.astype(np.uint64)) for r in qs]
    t0 = time.perf_counter()
    lists = []
    for m in qm:
        cand = host.query(m, 20)
        lists.append(sorted(cand, key=lambda d: (-m.jaccard(ms[d]), d))[:10])
    res["host_topk10_per_query_ms"] = round((time.perf_counter() - t0) * 1000 / len(qm), 4)
    got = small.query_topk(qs, 10)[0]
    res["host_equal"] = all(list(r[r >= 0]) == w for r, w in zip(got, lists))
    line = json.dumps(res)
    print(line)
    with open(a.out, "a") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
