"""GpuLSHEnsemble (containment search on the device) against the host MinHashLSHEnsemble.

    python tools/bench_ensemble.py [--sets 1000000] [--queries 100000] [--host-sets 20000] [--host-queries 1000]
                                   [--out profiles/h100_ensemble.jsonl]

Corpus: --sets token sets with heavy-tailed sizes (seeded), their K = 128 signatures built by the signature kernel.
Queries: subsets of indexed sets (a random share of one set's tokens: containment 1), supersets (an indexed set plus
random tokens) and unrelated sets.  The configuration is the default-like threshold 0.5, 16 partitions, m = 8.
Device: index() and query() with and without eq, CUDA events around the whole call after a warm-up, 3 rounds each;
index()'s host part (the reference's partitioning over the distinct sizes, the size order and the walk) is also timed
alone.
Host: this package's MinHashLSHEnsemble (dict buckets, a Python walk per query) indexes the first --host-sets sets and
answers --host-queries queries; a device index over the same sets answers the same queries and the outputs are compared.
Prints one JSON line and appends it to --out, with the card's name and power limit read in the same process.
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import datasketch_b200 as dsk  # noqa: E402
from datasketch_b200.lshensemble import _index_plan  # noqa: E402
from datasketch_b200.minhash import _make_permutations  # noqa: E402

THR, K, NUM_PART, M = 0.5, 128, 16, 8


def gpu_card():
    """The card's name, power limit and top SM clock, read in the same process as the timings beside them."""
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def corpus(n, nq, host_sets, host_queries, seed=0):
    """Token sets (CSR, int32 tokens) with heavy-tailed sizes, and queries with planted containment (the first
    host_queries of them built from the first host_sets sets, which the host index holds)."""
    rs = np.random.RandomState(seed)
    sizes = np.clip((rs.pareto(1.2, n) * 20 + 5).astype(np.int64), 5, 5000)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(sizes, out=off[1:])
    tok = rs.randint(-2 ** 31, 2 ** 31 - 1, size=int(off[-1]), dtype=np.int64).astype(np.int32)
    qsets = []
    for j in range(nq):
        src = int(rs.randint(host_sets if j < host_queries else n))
        s = tok[off[src]:off[src + 1]]
        kind = j % 4
        if kind < 2:                                                   # subset: containment 1
            qsets.append(s[:max(1, int(len(s) * rs.uniform(0.05, 1.0)))])
        elif kind == 2:                                                # superset
            extra = rs.randint(-2 ** 31, 2 ** 31 - 1, size=int(rs.randint(1, 4 * len(s) + 2)), dtype=np.int64)
            qsets.append(np.concatenate([s, extra.astype(np.int32)]))
        else:                                                          # unrelated
            qsets.append(rs.randint(-2 ** 31, 2 ** 31 - 1, size=int(sizes[rs.randint(n)]), dtype=np.int64).astype(np.int32))
    qsizes = np.array([len(q) for q in qsets], dtype=np.int64)
    qoff = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum(qsizes, out=qoff[1:])
    return tok, off, sizes, np.concatenate(qsets), qoff, qsizes


def signatures(tok, off, perms):
    d_tok = torch.from_numpy(tok).cuda()
    d_off = torch.from_numpy(off).cuda()
    sig = dsk.engine.bulk_signatures_device(d_tok, d_off, len(tok), perms)
    torch.cuda.synchronize()
    return sig


def ev(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def csr_sets(ptr, idx):
    return [set(idx[ptr[q]:ptr[q + 1]].tolist()) for q in range(len(ptr) - 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--host-sets", type=int, default=20_000)
    ap.add_argument("--host-queries", type=int, default=1_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ensemble.jsonl"))
    a = ap.parse_args()
    card = gpu_card()
    perms = _make_permutations(K, 1)
    hn, hq = min(a.host_sets, a.sets), min(a.host_queries, a.queries)
    tok, off, sizes, qtok, qoff, qsizes = corpus(a.sets, a.queries, hn, hq)
    sig = signatures(tok, off, perms)
    qsig = signatures(qtok, qoff, perms)
    res = {"config": "GpuLSHEnsemble(threshold=%g, num_perm=%d, num_part=%d, m=%d)" % (THR, K, NUM_PART, M),
           "sets": a.sets, "queries": a.queries, "tokens": int(off[-1]), "query_tokens": int(qoff[-1])}

    # -- device: index (a fresh object per round: index() is callable once) and query -----------------------------------
    warm = dsk.GpuLSHEnsemble(threshold=THR, num_perm=K, num_part=NUM_PART, m=M)
    warm.index(sig[:10_000], sizes[:10_000])
    warm.query(qsig[:1000], qsizes[:1000], with_eq=True)
    rs_ = sorted({int(r) for _, r in warm.params})
    res["rs"], res["sum_b_r"] = rs_, sum(K // r for r in rs_)
    res["index_bytes"] = int(dsk._native.load().dsk_lsh_ensemble_index_bytes(warm._h, a.sets))
    del warm
    index_ms, ens = [], None
    for _ in range(a.rounds):
        ens = None
        gc.collect()
        ens = dsk.GpuLSHEnsemble(threshold=THR, num_perm=K, num_part=NUM_PART, m=M)
        t, _ = ev(lambda: ens.index(sig, sizes))
        index_ms.append(t)
    res["index_ms"] = index_ms
    t0 = time.perf_counter()                                          # its host part: partitions, size order, walk
    _index_plan(sizes, NUM_PART)
    res["index_host_plan_s"] = time.perf_counter() - t0
    res["index_distinct_sizes"] = int(len(np.unique(sizes)))
    res["uppers"] = [None if u is None else int(u) for u in ens.uppers]
    ens.query(qsig, qsizes, to_host=False)
    ens.query(qsig, qsizes, with_eq=True, to_host=False)
    q_ms, qe_ms = [], []
    for _ in range(a.rounds):                                         # alternated
        t, out = ev(lambda: ens.query(qsig, qsizes, to_host=False))
        q_ms.append(t)
        t, out_eq = ev(lambda: ens.query(qsig, qsizes, with_eq=True, to_host=False))
        qe_ms.append(t)
    res["query_ms"], res["query_eq_ms"] = q_ms, qe_ms
    res["candidates"] = int(out[0][-1].item())
    res["queries_per_s"] = a.queries / (min(q_ms) / 1e3)
    res["eq_fill_identical_idx"] = bool(torch.equal(out[0], out_eq[0]) and torch.equal(out[1], out_eq[1]))
    del ens, out, out_eq
    gc.collect()

    # -- host comparison on a corpus the host can index ----------------------------------------------------------------
    hsig = sig[:hn].cpu().numpy().view(np.uint32)
    hq_sig = qsig[:hq].cpu().numpy().view(np.uint32)
    mhs = [dsk.MinHash(num_perm=K, seed=1, hashvalues=row.astype(np.uint64)) for row in hsig]
    qmhs = [dsk.MinHash(num_perm=K, seed=1, hashvalues=row.astype(np.uint64)) for row in hq_sig]
    host = dsk.MinHashLSHEnsemble(threshold=THR, num_perm=K, num_part=NUM_PART, m=M)
    t0 = time.perf_counter()
    host.index([(i, mhs[i], int(sizes[i])) for i in range(hn)])
    t_index = time.perf_counter() - t0
    t0 = time.perf_counter()
    want = [set(host.query(qmhs[q], int(qsizes[q]))) for q in range(hq)]
    t_query = time.perf_counter() - t0
    small = dsk.GpuLSHEnsemble(threshold=THR, num_perm=K, num_part=NUM_PART, m=M)
    t_dev_index, _ = ev(lambda: small.index(sig[:hn], sizes[:hn]))
    t_dev_query, got = ev(lambda: small.query(qsig[:hq], qsizes[:hq]))
    res.update({"host_sets": hn, "host_queries": hq, "host_index_s": t_index, "host_query_s": t_query,
                "host_us_per_set": t_index / hn * 1e6, "host_us_per_query": t_query / hq * 1e6,
                "device_small_index_ms": t_dev_index, "device_small_query_ms": t_dev_query,
                "host_candidates": sum(len(w) for w in want),
                "host_partitions_equal": [None if u is None else int(u) for u in host.uppers] ==
                [None if u is None else int(u) for u in small.uppers],
                "outputs_equal": csr_sets(*got) == want})
    line = dict(card, command="python tools/bench_ensemble.py " + " ".join(sys.argv[1:]), result=res)
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "a") as f:
        f.write(json.dumps(line) + "\n")
    if not res["outputs_equal"] or not res["host_partitions_equal"]:
        sys.exit("device and host outputs differ")


if __name__ == "__main__":
    main()
