"""GpuLSHEnsemble's containment estimates on the device against the torch flow a user would write on query()'s output.

    python tools/bench_ensemble_containment.py [--sets 1000000] [--queries 100000] [--rounds 3]
                                               [--out profiles/h100_ensemble_containment.jsonl]

Corpus, signatures and configuration (threshold 0.5, K = 128, 16 partitions, m = 8) are tools/bench_ensemble.py's.
Timed with CUDA events around whole calls, after a warm-up of each, alternated over --rounds rounds:
  * query_containment(0.8)  against query(with_eq=True, to_host=False) + torch: gather the candidates' sizes, the
                            estimate, the mask, the re-built CSR;
  * query_topk(10, 0.8)     against the same flow + a segmented sort by (-c, row) and the first 10 of each query;
  * containment_pairs(0.8)  against query() of all indexed rows with their own sizes + the same flow, minus self pairs.
Each pair of outputs is compared in the same run (rows, eq and the bits of c).  One quality line over the first 1,000
queries: mean |c - exact containment| from the token sets, and the precision and recall of c >= 0.8 among the candidates.
Prints one JSON line and appends it to --out, with the card's name, power limit and top SM clock read in the same process.
"""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
import datasketch_b200 as dsk  # noqa: E402
from bench_ensemble import K, M, NUM_PART, THR, corpus, ev, gpu_card, signatures  # noqa: E402
from datasketch_b200.minhash import _make_permutations  # noqa: E402

T, TOPK = 0.8, 10


def torch_filter(ptr, idx, eq, d_qsizes, d_sizes, t, drop_self=False):
    """query()'s CSR -> (ptr, idx, eq, c) of the candidates with c >= t (and, for the self-join, idx != row)."""
    seg = torch.repeat_interleave(torch.arange(len(ptr) - 1, device=ptr.device), ptr.diff())
    sq = d_qsizes[seg]
    j = eq.double() / K
    c = j * (sq + d_sizes[idx.long()]).double() / (sq.double() * (1 + j))
    keep = c >= t
    if drop_self:
        keep &= idx.long() != seg
    cm = torch.zeros(len(keep) + 1, dtype=torch.int64, device=ptr.device)
    torch.cumsum(keep, 0, out=cm[1:])
    return cm[ptr], idx[keep], eq[keep], c[keep]


def torch_topk(ptr, idx, eq, c, k):
    """The first k of each segment in the order (-c, row), padded with -1 / -1 / -1.0: three stable sorts."""
    nq = len(ptr) - 1
    seg = torch.repeat_interleave(torch.arange(nq, device=ptr.device), ptr.diff())
    o = torch.sort(idx, stable=True).indices
    o = o[torch.sort(-c[o], stable=True).indices]
    o = o[torch.sort(seg[o], stable=True).indices]
    pos = torch.arange(len(o), device=ptr.device) - ptr[seg[o]]
    take = pos < k
    out_i = torch.full((nq, k), -1, dtype=torch.int32, device=ptr.device)
    out_e = torch.full((nq, k), -1, dtype=torch.int32, device=ptr.device)
    out_c = torch.full((nq, k), -1.0, dtype=torch.float64, device=ptr.device)
    rows, cols, sel = seg[o][take], pos[take], o[take]
    out_i[rows, cols], out_e[rows, cols], out_c[rows, cols] = idx[sel], eq[sel], c[sel]
    return out_i, out_e, out_c


def same_csr(a, b):
    """Equal CSR results up to the order inside each segment: rows, eq and the bits of c."""
    if not torch.equal(a[0], b[0]):
        return False
    seg = torch.repeat_interleave(torch.arange(len(a[0]) - 1, device=a[0].device), a[0].diff())
    oa = torch.argsort(seg * (1 << 31) + a[1].long())
    ob = torch.argsort(seg * (1 << 31) + b[1].long())
    return all(torch.equal(x[oa].view(torch.int64) if x.dtype == torch.float64 else x[oa],
                           y[ob].view(torch.int64) if y.dtype == torch.float64 else y[ob]) for x, y in zip(a[1:], b[1:]))


def timed(fns, rounds):
    """Alternated rounds of each fn after one warm-up call each: {name: [ms]}, and each fn's last output."""
    outs = {name: fn() for name, fn in fns.items()}
    times = {name: [] for name in fns}
    for _ in range(rounds):
        for name, fn in fns.items():
            t, outs[name] = ev(fn)
            times[name].append(t)
    return times, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--quality-queries", type=int, default=1_000)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(ROOT), "profiles", "h100_ensemble_containment.jsonl"))
    a = ap.parse_args()
    card = gpu_card()
    perms = _make_permutations(K, 1)
    tok, off, sizes, qtok, qoff, qsizes = corpus(a.sets, a.queries, min(20_000, a.sets), min(1_000, a.queries))
    sig = signatures(tok, off, perms)
    qsig = signatures(qtok, qoff, perms)
    res = {"config": "GpuLSHEnsemble(threshold=%g, num_perm=%d, num_part=%d, m=%d)" % (THR, K, NUM_PART, M),
           "sets": a.sets, "queries": a.queries, "min_containment": T, "k": TOPK}
    ens = dsk.GpuLSHEnsemble(threshold=THR, num_perm=K, num_part=NUM_PART, m=M)
    ens.index(sig, sizes)
    d_sizes = torch.from_numpy(sizes).cuda()
    d_qsizes = torch.from_numpy(qsizes).cuda()

    def flow_query():
        return torch_filter(*ens.query(qsig, qsizes, with_eq=True, to_host=False), d_qsizes, d_sizes, T)

    times, outs = timed({"query_containment_ms": lambda: ens.query_containment(qsig, qsizes, T, to_host=False),
                         "torch_flow_ms": flow_query}, a.rounds)
    res["query_containment"] = dict(times, kept=int(outs["torch_flow_ms"][0][-1].item()),
                                    outputs_equal=same_csr(outs["query_containment_ms"], outs["torch_flow_ms"]))
    del outs
    times, outs = timed({"query_topk_ms": lambda: ens.query_topk(qsig, qsizes, TOPK, T, to_host=False),
                         "torch_flow_ms": lambda: torch_topk(*flow_query(), TOPK)}, a.rounds)
    res["query_topk"] = dict(times, outputs_equal=all(
        torch.equal(x.view(torch.int64) if x.dtype == torch.float64 else x,
                    y.view(torch.int64) if y.dtype == torch.float64 else y)
        for x, y in zip(outs["query_topk_ms"], outs["torch_flow_ms"])))
    del outs
    gc.collect()

    def flow_pairs():
        return torch_filter(*ens.query(sig, sizes, with_eq=True, to_host=False), d_sizes, d_sizes, T, drop_self=True)

    times, outs = timed({"containment_pairs_ms": lambda: ens.containment_pairs(T, to_host=False),
                         "torch_flow_ms": flow_pairs}, a.rounds)
    res["containment_pairs"] = dict(times, pairs=int(outs["torch_flow_ms"][0][-1].item()),
                                    outputs_equal=same_csr(outs["containment_pairs_ms"], outs["torch_flow_ms"]))
    del outs
    gc.collect()

    # -- quality of the estimate on a sample, against the exact containment of the token sets -------------------------
    nqq = min(a.quality_queries, a.queries)
    ptr, idx, eq, c = ens.query_containment(qsig[:nqq], qsizes[:nqq])
    err, tp, fp, fn = [], 0, 0, 0
    for q in range(nqq):
        qs = set(qtok[qoff[q]:qoff[q + 1]].tolist())
        for x, cv in zip(idx[ptr[q]:ptr[q + 1]].tolist(), c[ptr[q]:ptr[q + 1]].tolist()):
            exact = len(qs.intersection(tok[off[x]:off[x + 1]].tolist())) / len(qs)
            err.append(abs(cv - exact))
            tp += cv >= T and exact >= T
            fp += cv >= T and exact < T
            fn += cv < T and exact >= T
    res["quality"] = {"queries": nqq, "candidates": len(err), "mean_abs_error": float(np.mean(err)) if err else None,
                      "precision": tp / (tp + fp) if tp + fp else None, "recall": tp / (tp + fn) if tp + fn else None}
    line = dict(card, command="python tools/bench_ensemble_containment.py " + " ".join(sys.argv[1:]), result=res)
    print(json.dumps(line), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "a") as f:
        f.write(json.dumps(line) + "\n")
    if not all(res[key]["outputs_equal"] for key in ("query_containment", "query_topk", "containment_pairs")):
        sys.exit("device and torch outputs differ")


if __name__ == "__main__":
    main()
