"""Secondary workloads of BASELINE.json (configs[2..4]) on ONE GPU, with the oracle's CPU numbers beside them.
These are not bench.py lines; they are evidence for the other rows of SURVEY.md section 8.

    python tools/bench_configs.py [--c3-docs 2000000] [--c4-vecs 20000] [--c5-rows 100000]
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
from datasketch_b200.minhash import _make_permutations  # noqa: E402
from oracle import oracle_np as o  # noqa: E402


def ev_time(fn, iters=3, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def c3(n_docs, t=128, k=256, n_query=100_000, fused_leg=False, dedup_leg=False, remove_leg=False, query_jaccard_leg=False,
       insert_unique_leg=False, n_unique=100_000, topk_leg=False):
    """10M x 128 tokens, K=256 + LSH(0.8) insert + query (here n_docs on one GPU).  dedup_leg: also the self-join of
    the index (candidate_pairs, duplicate_clusters with and without min_jaccard=0.8) against the host flow it replaces.
    remove_leg: also removal of the duplicates from the index and its compaction (c3_remove).  query_jaccard_leg: also
    queries verified on the device against the two-step flow they replace (c3_query_jaccard).  topk_leg: also the ranked
    lists query_topk / neighbors against the flows they replace (c3_topk).  insert_unique_leg: also
    GpuLSH.insert_unique of a batch of n_unique fresh documents against the flow it replaces (c3_insert_unique); the index
    then has room for them (its bucket tables are the same size)."""
    perms = _make_permutations(k, 1)
    g = torch.Generator(device="cuda").manual_seed(3)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n_docs, t), dtype=torch.int32, device="cuda", generator=g)
    # plant near-duplicates: 10 % of documents copy another one with ~10 % tokens resampled
    ndup = n_docs // 10
    src = torch.randint(0, n_docs, (ndup,), device="cuda", generator=g)
    dst = torch.randint(0, n_docs, (ndup,), device="cuda", generator=g)
    tok[dst] = tok[src]
    mask = torch.rand((ndup, t), device="cuda", generator=g) < 0.1
    tok[dst] = torch.where(mask, torch.randint(-2 ** 31, 2 ** 31 - 1, (ndup, t), dtype=torch.int32, device="cuda", generator=g), tok[dst])
    off = torch.arange(0, (n_docs + 1) * t, t, dtype=torch.int64, device="cuda")
    sig = torch.empty((n_docs, k), dtype=torch.int32, device="cuda")
    ms_sig = ev_time(lambda: dsk.engine.bulk_signatures_device(tok.view(-1), off, n_docs * t, perms, d_out=sig))
    warm = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=4096)
    warm.insert(sig[:4096])                      # first launch of the kernels (module load, attribute set) is not timed
    warm.query(sig[:64], to_host=False)
    del warm
    lsh = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=n_docs + (n_unique if insert_unique_leg else 0))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    lsh.insert(sig)
    e1.record()
    torch.cuda.synchronize()
    ms_ins = e0.elapsed_time(e1)
    # fused: tokens -> signatures in the index's storage + bucket updates in ONE launch (GpuLSH.insert_tokens); three fresh
    # indexes, the first one warms the kernel up; candidates of the same queries must be identical to the two-step index
    ms_fused = []
    fused = None
    for rep in range(3 if fused_leg else 0):
        del fused
        fused = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=n_docs)
        torch.cuda.synchronize()
        e0.record()
        fused.insert_tokens(tok.view(-1), off, n_docs * t, perms)
        e1.record()
        torch.cuda.synchronize()
        ms_fused.append(e0.elapsed_time(e1))
    q = sig[torch.randint(0, n_docs, (n_query,), device="cuda", generator=g)]
    same = None
    if fused_leg:
        pf, xf = fused.query(q[:20_000], to_host=False)
        pp, xp = lsh.query(q[:20_000], to_host=False)
        same = bool(torch.equal(pf, pp)) and bool(torch.equal(
            torch.sort(xf.long() + torch.repeat_interleave(torch.arange(20_000, device="cuda"), pf[1:] - pf[:-1]) * n_docs)[0],
            torch.sort(xp.long() + torch.repeat_interleave(torch.arange(20_000, device="cuda"), pp[1:] - pp[:-1]) * n_docs)[0]))
        del fused
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ptr, idx = lsh.query(q, to_host=False)
    torch.cuda.synchronize()
    ms_q = (time.perf_counter() - t0) * 1e3
    # CPU oracle on a small sample: dict insert + query per document
    ns = 20_000
    hs = sig[:ns].cpu().numpy().view(np.uint32).astype(np.uint64)
    ref = o.DictLSH(k, lsh.b, lsh.r)
    t0 = time.perf_counter()
    for i, row in enumerate(hs):
        ref.insert(i, row, check_duplication=False)
    cpu_ins = (time.perf_counter() - t0) / ns
    t0 = time.perf_counter()
    for row in hs[:5000]:
        ref.query(row)
    cpu_q = (time.perf_counter() - t0) / 5000
    dedup = c3_dedup(lsh, src, dst, ref, hs) if dedup_leg else {}
    if remove_leg:
        dedup.update(c3_remove(lsh, sig, q))
    if query_jaccard_leg:
        dedup.update(c3_query_jaccard(lsh, sig, tok, perms))
    if topk_leg:
        dedup.update(c3_topk(lsh, tok, perms))
    if insert_unique_leg:
        dedup.update(c3_insert_unique(lsh, tok, perms, n_unique))
    return {"config": "C3 (1 GPU)", "docs": n_docs, "tokens": t, "num_perm": k, "b": lsh.b, "r": lsh.r,
            "signature_ms": ms_sig, "signatures_per_s": n_docs / ms_sig * 1e3,
            "lsh_insert_ms": ms_ins, "lsh_insert_docs_per_s": n_docs / ms_ins * 1e3,
            "fused_signatures_plus_insert_ms": min(ms_fused[1:]) if ms_fused else None, "fused_runs_ms": ms_fused,
            "two_step_signatures_plus_insert_ms": ms_sig + ms_ins, "fused_candidates_identical": same,
            "lsh_query_ms": ms_q, "queries": n_query, "lsh_queries_per_s": n_query / ms_q * 1e3,
            "candidates_total": int(ptr[-1].item()),
            "cpu_oracle_insert_us_per_doc": cpu_ins * 1e6, "cpu_oracle_query_us_per_doc": cpu_q * 1e6, **dedup}


def c3_dedup(lsh, src, dst, ref, hs, min_jaccard=0.8):
    """Self-join of the C3 index on the device, warmed up, timed with CUDA events; beside it, on the first len(hs)
    documents (already in the dict oracle ``ref``), the host flow it replaces: DictLSH.query per document, oracle_np.jaccard
    per pair, scipy connected components of the pairs with jaccard >= min_jaccard."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    n = len(lsh)
    ms_pairs = ev_time(lambda: lsh.candidate_pairs(to_host=False))
    ms_cl = ev_time(lambda: lsh.duplicate_clusters(to_host=False))
    ms_cl_t = ev_time(lambda: lsh.duplicate_clusters(min_jaccard, to_host=False))
    ptr, _, _ = lsh.candidate_pairs(to_host=False)
    pairs = int(ptr[-1].item())
    out = {"dedup_pairs": pairs, "dedup_candidate_pairs_ms": ms_pairs, "dedup_pairs_per_s": pairs / ms_pairs * 1e3,
           "dedup_candidate_pairs_docs_per_s": n / ms_pairs * 1e3,
           "dedup_clusters_ms": ms_cl, "dedup_clusters_docs_per_s": n / ms_cl * 1e3,
           "dedup_min_jaccard": min_jaccard, "dedup_clusters_min_jaccard_ms": ms_cl_t,
           "dedup_clusters_min_jaccard_docs_per_s": n / ms_cl_t * 1e3}
    ar = torch.arange(n, dtype=torch.int32, device="cuda")
    for tag, t in (("", None), ("_min_jaccard", min_jaccard)):
        labels = lsh.duplicate_clusters(t, to_host=False)
        out["dedup_clusters" + tag] = int((labels == ar).sum().item())
        out["dedup_planted_together" + tag] = float((labels[src] == labels[dst]).float().mean().item())
    t0 = time.perf_counter()
    ii, dd = [], []
    for i, row in enumerate(hs):
        for d in ref.query(row):
            if d < i and o.jaccard(row, hs[d]) >= min_jaccard:
                ii.append(i)
                dd.append(d)
    ns = len(hs)
    connected_components(coo_matrix((np.ones(len(ii)), (ii, dd)), shape=(ns, ns)), directed=False)
    out["dedup_host_flow_us_per_doc"] = (time.perf_counter() - t0) / ns * 1e6
    return out


def c3_remove(lsh, sig, q, min_jaccard=0.8, rounds=3):
    """GpuLSH.remove of the non-root documents of duplicate_clusters(min_jaccard), then the walks with removals present,
    then compact().  The removals go to a second index of the same rows, so that the calls without removals (``lsh``, the
    kernels that run when nothing was removed) and with them (the removal-aware kernels) alternate in one process: each
    round times every call on both indexes with CUDA events (3 calls after 1 warm-up call).  remove() and compact() run
    once each, so they are timed once: both wait for the device inside (remove() checks its ids first, compact() reads
    the number of remaining documents), and the events span the whole call."""
    n, k = len(lsh), lsh.h
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rm = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=n)
    torch.cuda.synchronize()
    e0.record()
    rm.insert(sig)
    e1.record()
    torch.cuda.synchronize()
    ms_insert = e0.elapsed_time(e1)
    labels = rm.duplicate_clusters(min_jaccard, to_host=False)
    gone = torch.nonzero(labels != torch.arange(n, dtype=torch.int32, device="cuda")).view(-1)
    small = dsk.GpuLSH(threshold=0.8, num_perm=k, capacity=64)   # first launch of the remove / alive kernels: not timed
    small.insert(sig[:64])
    small.remove([1, 2])
    del small
    torch.cuda.synchronize()
    e0.record()
    rm.remove(gone)
    e1.record()
    torch.cuda.synchronize()
    ms_remove = e0.elapsed_time(e1)
    calls = {"query": lambda ix: ix.query(q, to_host=False),
             "candidate_pairs": lambda ix: ix.candidate_pairs(to_host=False),
             "duplicate_clusters": lambda ix: ix.duplicate_clusters(to_host=False),
             "duplicate_clusters_min_jaccard": lambda ix: ix.duplicate_clusters(min_jaccard, to_host=False)}
    times = {name: {"without": [], "with": []} for name in calls}
    for _ in range(rounds):
        for name, fn in calls.items():
            times[name]["without"].append(ev_time(lambda: fn(lsh)))
            times[name]["with"].append(ev_time(lambda: fn(rm)))
    p0, x0, _ = lsh.candidate_pairs(to_host=False)
    rows0 = torch.repeat_interleave(torch.arange(n, device="cuda"), p0[1:] - p0[:-1])
    alive = rm.alive(to_host=False)
    kept_pairs = int((alive[rows0] & alive[x0.long()]).sum().item())
    p1, _, _ = rm.candidate_pairs(to_host=False)
    torch.cuda.synchronize()
    e0.record()
    remap = rm.compact(to_host=False)
    e1.record()
    torch.cuda.synchronize()
    ms_compact = e0.elapsed_time(e1)
    ms_pairs_after = ev_time(lambda: rm.candidate_pairs(to_host=False))
    p2, _, _ = rm.candidate_pairs(to_host=False)
    out = {"remove_min_jaccard": min_jaccard, "remove_docs": int(gone.numel()), "remove_ms_once": ms_remove,
           "remove_second_index_insert_ms": ms_insert, "remove_docs_remaining": len(rm),
           "remove_pairs_before": int(p0[-1].item()), "remove_pairs_with_removals": int(p1[-1].item()),
           "remove_pairs_among_remaining_before": kept_pairs, "remove_pairs_after_compact": int(p2[-1].item()),
           "remove_remap_monotone": bool((remap[remap >= 0].diff() == 1).all().item()),
           "remove_compact_ms_once": ms_compact, "remove_candidate_pairs_after_compact_ms": ms_pairs_after}
    for name, t in times.items():
        out["remove_%s_ms_without_removals" % name] = t["without"]
        out["remove_%s_ms_with_removals" % name] = t["with"]
    return out


def gpu_card():
    """The card's name, power limit and top SM clock, read in the same process as the timings beside them."""
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def c3_fresh_queries(n, tok, perms, n_query):
    """Signatures of n_query fresh documents against the first n rows of `tok`: half of them copies of indexed documents
    with 10 % of the tokens resampled, half unrelated, built by the same signature kernel (the same rows on every call)."""
    t = tok.shape[1]
    g = torch.Generator(device="cuda").manual_seed(11)
    qtok = torch.randint(-2 ** 31, 2 ** 31 - 1, (n_query, t), dtype=torch.int32, device="cuda", generator=g)
    h = n_query // 2
    src = torch.randint(0, n, (h,), device="cuda", generator=g)
    qtok[:h] = torch.where(torch.rand((h, t), device="cuda", generator=g) < 0.1, qtok[:h], tok[src])
    qoff = torch.arange(0, (n_query + 1) * t, t, dtype=torch.int64, device="cuda")
    return dsk.engine.bulk_signatures_device(qtok.view(-1), qoff, n_query * t, perms)


def c3_query_jaccard(lsh, sig, tok, perms, n_query=100_000, min_jaccard=0.8, rounds=3):
    """GpuLSH.query_jaccard / query_best for n_query fresh documents against the C3 index: half of them copies of indexed
    documents with 10 % of the tokens resampled, half unrelated, their signatures built by the same kernel.  Beside them,
    query() and the two-step flow they replace: query, the (query, document) pairs expanded with repeat_interleave,
    codec.jaccard_pairs on cat([index rows, queries]) and the filter re-packed as CSR.  Each round times every call with
    CUDA events (3 calls after 1 warm-up call), the calls alternating; the outputs are compared in the same run."""
    n, k = len(lsh), lsh.h
    qs = c3_fresh_queries(n, tok, perms, n_query)
    ar = torch.arange(n_query, device="cuda")

    def two_step(thr):
        p, x = lsh.query(qs, to_host=False)
        rows = torch.repeat_interleave(ar, p[1:] - p[:-1])
        jac = dsk.codec.jaccard_pairs(torch.cat([sig, qs]), rows + n, x.long())
        keep = torch.from_numpy(jac >= thr).cuda()
        cnt = torch.from_numpy(np.rint(jac * k).astype(np.int32)).cuda()
        ptr = torch.zeros(n_query + 1, dtype=torch.int64, device="cuda")
        ptr[1:] = torch.cumsum(torch.bincount(rows[keep], minlength=n_query), 0)
        return ptr, x[keep], cnt[keep]

    calls = {"query": lambda: lsh.query(qs, to_host=False),
             "query_jaccard": lambda: lsh.query_jaccard(qs, to_host=False),
             "query_jaccard_min_jaccard": lambda: lsh.query_jaccard(qs, min_jaccard, to_host=False),
             "query_best_min_jaccard": lambda: lsh.query_best(qs, min_jaccard, to_host=False),
             "two_step_min_jaccard": lambda: two_step(min_jaccard)}
    times = {name: [] for name in calls}
    for _ in range(rounds):
        for name, fn in calls.items():
            times[name].append(ev_time(fn))
    # outputs: query_jaccard(min_jaccard) == the two-step flow (same sets, same eq); query_best == their per-query argmax
    p1, x1, e1 = lsh.query_jaccard(qs, min_jaccard, to_host=False)
    p2, x2, e2 = two_step(min_jaccard)
    def keyed(p, x, e):
        key = torch.repeat_interleave(ar, p[1:] - p[:-1]) * n + x.long()
        order = torch.argsort(key)
        return key[order], e[order]
    k1, f1 = keyed(p1, x1, e1)
    k2, f2 = keyed(p2, x2, e2)
    same = bool(torch.equal(p1, p2)) and bool(torch.equal(k1, k2)) and bool(torch.equal(f1, f2))
    rows = torch.repeat_interleave(ar, p2[1:] - p2[:-1])
    score = e2.long() * (1 << 32) - x2.long()                # largest eq, then smallest document
    top = torch.full((n_query,), -(1 << 62), dtype=torch.int64, device="cuda").scatter_reduce(0, rows, score, "amax")
    w_eq = torch.where(top > -(1 << 62), (top + (1 << 32) - 1) >> 32, torch.full_like(top, -1))
    w_idx = torch.where(w_eq >= 0, w_eq * (1 << 32) - top, torch.full_like(top, -1))
    bi, bq = lsh.query_best(qs, min_jaccard, to_host=False)
    best_same = bool(torch.equal(bi.long(), w_idx)) and bool(torch.equal(bq.long(), w_eq))
    p0, _ = lsh.query(qs, to_host=False)
    pa, _, _ = lsh.query_jaccard(qs, to_host=False)
    out = {"qj_queries": n_query, "qj_min_jaccard": min_jaccard, "qj_candidates": int(p0[-1].item()),
           "qj_candidates_unfiltered_equal_query": bool(torch.equal(p0, pa)), "qj_kept": int(p1[-1].item()),
           "qj_queries_with_best": int((bi >= 0).sum().item()),
           "qj_fused_equals_two_step": same, "qj_best_equals_two_step_argmax": best_same}
    for name, ts in times.items():
        out["qj_%s_ms" % name] = ts
    out.update({"qj_" + key: v for key, v in gpu_card().items()})
    return out


def segmented_topk(rows, idx, eq, n_rows, n_idx, k, num_perm):
    """(row, idx, eq) triples on the device -> ``[n_rows, k]`` idx / eq, per row sorted by larger eq, then smaller idx, cut
    at k and padded with -1: one torch sort of a combined int64 key (row, num_perm - eq, idx), then the rank in the row."""
    key = (rows.long() * (num_perm + 1) + (num_perm - eq.long())) * n_idx + idx.long()
    key, order = torch.sort(key)
    rows, idx, eq = rows[order].long(), idx[order], eq[order]
    start = torch.searchsorted(rows, torch.arange(n_rows, device=rows.device))
    rank = torch.arange(len(rows), device=rows.device) - start[rows]
    sel = rank < k
    oi = torch.full((n_rows, k), -1, dtype=torch.int32, device=rows.device)
    oe = torch.full((n_rows, k), -1, dtype=torch.int32, device=rows.device)
    oi[rows[sel], rank[sel]] = idx[sel].int()
    oe[rows[sel], rank[sel]] = eq[sel].int()
    return oi, oe


def c3_topk(lsh, tok, perms, n_query=100_000, k=10, min_jaccard=0.5, best_jaccard=0.8, rounds=3):
    """GpuLSH.query_topk / neighbors on the C3 index, each beside the flow it replaces: query_topk(k, min_jaccard) of
    n_query fresh documents (built as in c3_query_jaccard) against query_jaccard(min_jaccard) + a torch segmented top-k,
    query_topk(1, best_jaccard) against query_best(best_jaccard), and neighbors(k, min_jaccard) against
    candidate_pairs(min_jaccard) made symmetric + the same top-k.  Each round times every call with CUDA events (3 calls
    after 1 warm-up call), the calls alternating; the outputs are compared in the same run."""
    n, K = len(lsh), lsh.h
    qs = c3_fresh_queries(n, tok, perms, n_query)
    ar_q, ar_n = torch.arange(n_query, device="cuda"), torch.arange(n, device="cuda")

    def query_flow():
        p, x, e = lsh.query_jaccard(qs, min_jaccard, to_host=False)
        return segmented_topk(torch.repeat_interleave(ar_q, p[1:] - p[:-1]), x, e, n_query, n, k, K)

    def neighbors_flow():
        p, x, e = lsh.candidate_pairs(min_jaccard, to_host=False)
        i = torch.repeat_interleave(ar_n, p[1:] - p[:-1])
        return segmented_topk(torch.cat([i, x.long()]), torch.cat([x, i.int()]), torch.cat([e, e]), n, n, k, K)

    calls = {"query_topk": lambda: lsh.query_topk(qs, k, min_jaccard, to_host=False),
             "query_jaccard_torch_topk": query_flow,
             "query_topk_1": lambda: lsh.query_topk(qs, 1, best_jaccard, to_host=False),
             "query_best": lambda: lsh.query_best(qs, best_jaccard, to_host=False),
             "neighbors": lambda: lsh.neighbors(k, min_jaccard, to_host=False),
             "candidate_pairs_symmetric_torch_topk": neighbors_flow}
    times = {name: [] for name in calls}
    for _ in range(rounds):
        for name, fn in calls.items():
            times[name].append(ev_time(fn))
    qi, qe = lsh.query_topk(qs, k, min_jaccard, to_host=False)
    fi, fe = query_flow()
    ti, te = lsh.query_topk(qs, 1, best_jaccard, to_host=False)
    bi, be = lsh.query_best(qs, best_jaccard, to_host=False)
    ni, ne = lsh.neighbors(k, min_jaccard, to_host=False)
    si, se = neighbors_flow()
    p, _, _ = lsh.query_jaccard(qs, min_jaccard, to_host=False)
    pp, _, _ = lsh.candidate_pairs(min_jaccard, to_host=False)
    out = {"tk_queries": n_query, "tk_k": k, "tk_min_jaccard": min_jaccard, "tk_best_min_jaccard": best_jaccard,
           "tk_query_candidates_kept": int(p[-1].item()), "tk_queries_with_a_match": int((qi[:, 0] >= 0).sum().item()),
           "tk_query_entries": int((qi >= 0).sum().item()), "tk_pairs_kept": int(pp[-1].item()),
           "tk_docs_with_a_neighbor": int((ni[:, 0] >= 0).sum().item()), "tk_neighbor_entries": int((ni >= 0).sum().item()),
           "tk_query_topk_equals_flow": bool(torch.equal(qi, fi) and torch.equal(qe, fe)),
           "tk_query_topk_1_equals_query_best": bool(torch.equal(ti[:, 0], bi) and torch.equal(te[:, 0], be)),
           "tk_neighbors_equals_flow": bool(torch.equal(ni, si) and torch.equal(ne, se))}
    for name, ts in times.items():
        out["tk_%s_ms" % name] = ts
    out.update({"tk_" + key: v for key, v in gpu_card().items()})
    return out


def c3_unique_batch(tok, nb, g, chain=5, drift=0.05):
    """nb fresh token rows for a dedup batch against the documents `tok`: 40 % copies of indexed documents with 10 % of
    the tokens resampled, 20 % unrelated, 20 % drift chains of `chain` rows (each row its predecessor with `drift` of the
    tokens resampled) and 20 % exact copies of earlier rows of the batch, in that order."""
    n, t = tok.shape
    out = torch.randint(-2 ** 31, 2 ** 31 - 1, (nb, t), dtype=torch.int32, device="cuda", generator=g)
    a, b = int(nb * 0.4), int(nb * 0.2)
    c = int(nb * 0.2) // chain * chain
    src = torch.randint(0, n, (a,), device="cuda", generator=g)
    out[:a] = torch.where(torch.rand((a, t), device="cuda", generator=g) < 0.1, out[:a], tok[src])
    s0 = a + b                                                  # chain i holds rows s0 + i * chain + 0 .. chain - 1
    for step in range(1, chain):
        cur = out[s0 + step:s0 + c:chain]
        prev = out[s0 + step - 1:s0 + c:chain]
        out[s0 + step:s0 + c:chain] = torch.where(torch.rand(cur.shape, device="cuda", generator=g) < drift, cur, prev)
    csrc = torch.randint(0, a + b + c, (nb - a - b - c,), device="cuda", generator=g)
    out[a + b + c:] = out[csrc]
    return out


def two_step_unique(lsh, bsig, min_jaccard):
    """The flow GpuLSH.insert_unique replaces: query_best of the batch against the index, a temporary GpuLSH over the
    batch and its candidate_pairs(min_jaccard), the greedy loop over those pairs on the host, then insert of the kept
    rows.  Returns (kept, match, eq) as insert_unique does."""
    n0, nb = len(lsh), bsig.shape[0]
    bi, bq = lsh.query_best(bsig, min_jaccard)
    tmp = dsk.GpuLSH(num_perm=lsh.h, params=(lsh.b, lsh.r), capacity=max(nb, 1))
    tmp.insert(bsig)
    ptr, idx, eq = tmp.candidate_pairs(min_jaccard)
    del tmp
    ptr, idx, eq = ptr.tolist(), idx.tolist(), eq.tolist()
    kept = np.zeros(nb, dtype=bool)
    rank = np.full(nb, -1, dtype=np.int64)
    match, best = bi.astype(np.int64), bq.astype(np.int64)
    m = 0
    for j in range(nb):
        d_best, e_best, hit = int(match[j]), int(best[j]), match[j] >= 0
        for p in range(ptr[j], ptr[j + 1]):
            d = idx[p]
            if kept[d]:
                hit = True
                c, e = n0 + int(rank[d]), eq[p]
                if e > e_best or (e == e_best and c < d_best):
                    d_best, e_best = c, e
        if hit:
            match[j], best[j] = d_best, e_best
        else:
            kept[j], rank[j], m = True, m, m + 1
            match[j], best[j] = -1, -1
    if m:
        lsh.insert(bsig[torch.from_numpy(kept).to(bsig.device)])
    return kept, match.astype(np.int32), best.astype(np.int32)


def c3_insert_unique(lsh, tok, perms, nb, min_jaccard=0.8, rounds=3):
    """GpuLSH.insert_unique(min_jaccard) of nb fresh documents (c3_unique_batch) against the C3 index, beside the flow it
    replaces (two_step_unique), wall-clock from a synchronised device to the result, the two alternating.  After each
    call the kept rows are removed again and the index compacted (not timed).  In the same run the kept masks, matches
    and the indexes after either flow (query of a sample of the batch) are compared."""
    n, k = len(lsh), lsh.h
    t = tok.shape[1]
    g = torch.Generator(device="cuda").manual_seed(13)
    btok = c3_unique_batch(tok, nb, g)
    boff = torch.arange(0, (nb + 1) * t, t, dtype=torch.int64, device="cuda")
    bsig = dsk.engine.bulk_signatures_device(btok.view(-1), boff, nb * t, perms)
    probe = bsig[::25]

    def undo():
        if len(lsh) > n:
            lsh.remove(torch.arange(n, len(lsh), device="cuda"))
            lsh.compact()

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, res

    calls = {"insert_unique": lambda: lsh.insert_unique(bsig, min_jaccard),
             "two_step": lambda: two_step_unique(lsh, bsig, min_jaccard)}
    times = {name: [] for name in calls}
    results, states = {}, {}
    for rep in range(rounds + 1):                          # the first round warms both flows up
        for name, fn in calls.items():
            ms, res = timed(fn)
            if rep:
                times[name].append(ms)
            results[name] = res
            p, x = lsh.query(probe)
            states[name] = (p, [sorted(x[p[q]:p[q + 1]].tolist()) for q in range(len(p) - 1)], len(lsh))
            undo()
    (k1, m1, e1), (k2, m2, e2) = results["insert_unique"], results["two_step"]
    out = {"iu_batch": nb, "iu_min_jaccard": min_jaccard, "iu_index_docs": n, "iu_kept": int(k1.sum()),
           "iu_dropped_by_index": int(((m1 >= 0) & (m1 < n)).sum()), "iu_dropped_by_batch": int((m1 >= n).sum()),
           "iu_kept_equal": bool(np.array_equal(k1, k2)),
           "iu_match_eq_equal": bool(np.array_equal(m1, m2) and np.array_equal(e1, e2)),
           "iu_index_after_equal": bool(np.array_equal(states["insert_unique"][0], states["two_step"][0]) and
                                        states["insert_unique"][1:] == states["two_step"][1:])}
    for name, ts in times.items():
        out["iu_%s_ms" % name] = ts
    out.update({"iu_" + key: v for key, v in gpu_card().items()})
    return out


def c4(n_vec, dim=4096, ss=128):
    gen = dsk.WeightedMinHashGenerator(dim, ss, 1)
    g = torch.Generator(device="cuda").manual_seed(4)
    v = torch.rand((n_vec, dim), device="cuda", generator=g) * 10
    v[:, ::7] = 0
    gen.minhash_batch(v[:8])  # create the handle
    from datasketch_b200 import _native as nv
    h = gen._handle(0)
    out = torch.empty((n_vec, ss, 2), dtype=torch.int64, device="cuda")
    st = torch.empty((n_vec,), dtype=torch.int32, device="cuda")
    ms = ev_time(lambda: nv.check(nv.load().dsk_wmh_minhash(h, v.data_ptr(), n_vec, out.data_ptr(), st.data_ptr(), 0,
                                                             torch.cuda.current_stream().cuda_stream)), iters=2)
    par = o.wmh_params(dim, ss, 1)
    vs = v[:20].cpu().numpy()
    t0 = time.perf_counter()
    want = np.stack([o.wmh_minhash(x, *par) for x in vs])
    cpu = (time.perf_counter() - t0) / len(vs)
    got = out[:20].cpu().numpy()
    return {"config": "C4", "vectors": n_vec, "dim": dim, "sample_size": ss, "ms": ms,
            "vectors_per_s": n_vec / ms * 1e3, "evals_per_s": n_vec * dim * ss / ms * 1e3,
            "cpu_oracle_ms_per_vector": cpu * 1e3, "sampled_rows_identical": bool(np.array_equal(got, want)),
            "sampled_mismatching_samples": int((got != want).any(axis=2).sum())}


def c5(n_rows, k=128, topk=10):
    """All-pairs top-k: the exact kernel and the fingerprint-prefilter variant on the same matrix (identical lists
    required), on signatures without similarity (the C2 shape: every count is 0, ties by index) plus planted duplicates."""
    g = torch.Generator(device="cuda").manual_seed(5)
    sig = torch.randint(-2 ** 31, 2 ** 31 - 1, (n_rows, k), dtype=torch.int32, device="cuda", generator=g)
    sig[1::2][: n_rows // 4] = sig[0::2][: n_rows // 4]       # planted duplicates
    res = {}
    for name, pf in (("exact", False), ("prefilter", True)):
        dsk.codec.jaccard_topk(sig[:256], sig[:4096], topk=topk, self_base=0, to_host=False, prefilter=pf)   # first launch
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res[name] = dsk.codec.jaccard_topk(sig, sig, topk=topk, self_base=0, to_host=False, prefilter=pf)
        e1.record()
        torch.cuda.synchronize()
        res[name + "_ms"] = e0.elapsed_time(e1)
    same = bool(torch.equal(res["exact"][0], res["prefilter"][0]) and torch.equal(res["exact"][1], res["prefilter"][1]))
    # brute-force check of sampled rows
    rows = torch.linspace(0, n_rows - 1, 64, device="cuda").long()
    cnts = (sig[rows][:, None, :] == sig[None, :, :]).sum(dim=2)
    cnts[torch.arange(len(rows)), rows] = -1
    wrong = 0
    for i, r in enumerate(rows.tolist()):
        c = cnts[i]
        order = torch.argsort(-c * (n_rows + 1) + torch.arange(n_rows, device="cuda"))[:topk]   # count desc, index asc
        wrong += int(not torch.equal(order, res["prefilter"][1][r]))
    a = sig[:2000].cpu().numpy().view(np.uint32).astype(np.uint64)
    t0 = time.perf_counter()
    for i in range(0, 2000, 2):
        o.jaccard(a[i], a[i + 1])
    cpu = (time.perf_counter() - t0) / 1000
    ms = res["prefilter_ms"]
    return {"config": "C5 (1 GPU)", "rows": n_rows, "num_perm": k, "topk": topk, "ms": ms, "ms_exact_kernel": res["exact_ms"],
            "speedup_vs_exact_kernel": res["exact_ms"] / ms, "lists_identical_to_exact_kernel": same, "rows_wrong": wrong,
            "pairs_per_s": n_rows * n_rows / ms * 1e3, "compares_per_s": n_rows * n_rows * k / ms * 1e3,
            "cpu_oracle_us_per_pair": cpu * 1e6}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--c3-docs", type=int, default=2_000_000)
    ap.add_argument("--c4-vecs", type=int, default=20_000)
    ap.add_argument("--c5-rows", type=int, default=100_000)
    ap.add_argument("--c3-fused", action="store_true",
                    help="also time GpuLSH.insert_tokens (fused signatures + insert); tools/diag_fused.py times it alone")
    ap.add_argument("--c3-dedup", action="store_true",
                    help="also time GpuLSH.candidate_pairs / duplicate_clusters on the C3 index and the host flow they replace")
    ap.add_argument("--c3-remove", action="store_true",
                    help="after the dedup leg: GpuLSH.remove of the duplicates, the walks with removals present beside the "
                         "same calls without removals, and compact()")
    ap.add_argument("--c3-query-jaccard", action="store_true",
                    help="also time GpuLSH.query_jaccard / query_best for 100k fresh documents against the C3 index, beside "
                         "query() and the two-step flow they replace, and compare their outputs")
    ap.add_argument("--c3-insert-unique", action="store_true",
                    help="also time GpuLSH.insert_unique(0.8) of 100k fresh documents against the C3 index, beside the "
                         "flow it replaces (query_best, a temporary index's candidate_pairs, a host greedy loop, insert), "
                         "and compare their outputs")
    ap.add_argument("--c3-topk", action="store_true",
                    help="also time GpuLSH.query_topk(10, 0.5) / query_topk(1, 0.8) for 100k fresh documents and "
                         "neighbors(10, 0.5) on the C3 index, beside the flows they replace (query_jaccard + a torch "
                         "segmented top-k, query_best, symmetrised candidate_pairs + the same top-k), and compare outputs")
    a = ap.parse_args()
    if a.c3_docs > 0:
        print(json.dumps(c3(a.c3_docs, fused_leg=a.c3_fused, dedup_leg=a.c3_dedup, remove_leg=a.c3_remove,
                            query_jaccard_leg=a.c3_query_jaccard, insert_unique_leg=a.c3_insert_unique,
                            topk_leg=a.c3_topk)), flush=True)
    for fn, arg in ((c4, a.c4_vecs), (c5, a.c5_rows)):
        if arg > 0:
            print(json.dumps(fn(arg)), flush=True)
