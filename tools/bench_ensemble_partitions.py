"""The size partitioner of GpuLSHEnsemble.index on the device (optimal_partitions_device) against the host optimal_partitions.

    python tools/bench_ensemble_partitions.py [--d 1000 3550 10000 20000] [--num-part 16] [--host-max-d 3550]
                                              [--rounds 3] [--out profiles/h100_ensemble_partitions.jsonl]

Distributions: D = 3550 is the distinct set sizes of tools/bench_ensemble.py's 1M-set corpus (the same seeded size draw)
with their counts; every other D is D distinct sizes drawn log-uniformly up to 10^9 with heavy-tailed (Pareto) counts.
Device: one warm-up call, then --rounds calls, each timed with CUDA events around the whole call (the copies of sizes and
counts, the cost triangle, the dynamic programme, the back-tracking, the copy back and the synchronisation; the workspace
comes from torch's caching allocator).  Host: optimal_partitions once for D <= --host-max-d; the bounds must be equal.
For the corpus of D = 3550 it also times _index_plan with the device partitioner (np.unique, the partitioner, the stable
argsort of the 1M sizes and the walk) and reports the share that is not the partitioner.
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
from datasketch_b200 import _native as nv  # noqa: E402
from datasketch_b200.lshensemble import _index_plan, optimal_partitions, optimal_partitions_device  # noqa: E402


def gpu_card():
    """The card's name, power limit and top SM clock, read in the same process as the timings beside them."""
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def corpus_sizes(n=1_000_000, seed=0):
    """The per-set sizes of tools/bench_ensemble.py's corpus (its first draw from the same seed)."""
    rs = np.random.RandomState(seed)
    return np.clip((rs.pareto(1.2, n) * 20 + 5).astype(np.int64), 5, 5000)


def distribution(d, seed):
    rs = np.random.RandomState(seed)
    sizes = np.unique(np.exp(rs.uniform(0, np.log(1e9), 3 * d)).astype(np.int64) + 1)
    sizes = np.sort(rs.choice(sizes, d, replace=False))
    counts = np.minimum((rs.pareto(1.0, d) * 5 + 1).astype(np.int64), 10 ** 7)
    return sizes, counts


def ev(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, nargs="+", default=[1000, 3550, 10000, 20000])
    ap.add_argument("--num-part", type=int, default=16)
    ap.add_argument("--host-max-d", type=int, default=3550)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ensemble_partitions.jsonl"))
    a = ap.parse_args()
    card = gpu_card()
    k = a.num_part
    cs = corpus_sizes()
    runs, all_equal = [], True
    for d in a.d:
        if d == 3550:
            sizes, counts = np.unique(cs, return_counts=True)
            assert len(sizes) == 3550, len(sizes)
            source = "tools/bench_ensemble.py corpus"
        else:
            sizes, counts = distribution(d, d)
            source = "log-uniform sizes up to 1e9, Pareto counts"
        ws = int(nv.load().dsk_ensemble_partition_workspace_size(d, k))
        optimal_partitions_device(sizes, counts, k)                    # warm-up
        dev_ms, got = [], None
        for _ in range(a.rounds):
            t, got = ev(lambda: optimal_partitions_device(sizes, counts, k))
            dev_ms.append(t)
        r = {"d": d, "num_part": k, "sizes": source, "workspace_bytes": ws, "additions": d * (d + 1) * (d + 2) // 6,
             "divisions": d * (d + 1) // 2, "device_ms": dev_ms, "uppers": [int(u) for _, u in got]}
        if d <= a.host_max_d:
            t0 = time.perf_counter()
            want = optimal_partitions(sizes, counts, k)
            r["host_s"] = time.perf_counter() - t0
            r["bounds_equal"] = [(int(x), int(y)) for x, y in got] == [(int(x), int(y)) for x, y in want]
            all_equal = all_equal and r["bounds_equal"]
        if d == 3550:
            part = lambda s, c, kk: optimal_partitions_device(s, c, kk)   # noqa: E731
            _index_plan(cs, k, part)
            plan = []
            for _ in range(a.rounds):
                t0 = time.perf_counter()
                _index_plan(cs, k, part)
                plan.append((time.perf_counter() - t0) * 1e3)
            r["index_plan_ms"] = plan
            r["index_plan_other_ms"] = min(plan) - min(dev_ms)          # np.unique, argsort, walk
        runs.append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    line = dict(card, command="python tools/bench_ensemble_partitions.py " + " ".join(sys.argv[1:]), result=runs)
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "a") as f:
        f.write(json.dumps(line) + "\n")
    if not all_equal:
        sys.exit("device and host partitions differ")


if __name__ == "__main__":
    main()
