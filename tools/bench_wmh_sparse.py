"""Weighted MinHash on sparse rows (dsk_wmh_minhash_csr, DESIGN.md section 4l) against the densified path.

    python tools/bench_wmh_sparse.py [--rows 1000000] [--nnz 200] [--out profiles/h100_wmh_sparse.jsonl]

Workloads (sample size 128, seed 1; corpora seeded and built on the device):
  a  dim 2^20, --rows rows of about --nnz entries, Zipf-like columns (a Pareto(0.1) draw folded into [0, dim), so the
     low columns are hot), integer weights 1..49: CSR kernel time, rows/s, parameter-gather bytes/s
     (nnz x 3 x 4 x ss_pad) as a share of the data-sheet 3.35 TB/s, evaluations/s; end-to-end minhash_batch of the
     same matrix as scipy CSR (host log, copies both ways included).
  b  the same shape with uniform columns (the least L2 reuse).
  c  dim 4096 at 50 % density, 100k rows: the CSR kernel against the dense kernel on the densified rows, and
     minhash_batch(scipy CSR) against minhash_batch(X.toarray()) end to end.
  d  the sparse minhash_many as it was (rows densified in 256 MB slabs, dense kernel) on 1,024 rows of (a), per row,
     against minhash_many now.
  e  (a)'s rows plus one row of 10^6 entries.
Kernel times: CUDA events around one launch, after a warm-up launch, --repeats times.  In every workload sampled rows
are compared with the dense kernel (dsk_wmh_minhash) on the same rows densified, in the same run.  Prints one JSON line
and appends it to --out, with the card's name and power limit read in the same process.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import datasketch_b200 as dsk  # noqa: E402
from datasketch_b200 import _native as nv  # noqa: E402

SS = 128
SS_PAD = 128
HBM_BYTES_PER_S = 3.35e12
WMH_MANY, WMH_INPUT_LOG = 1, 2


def gpu_card():
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def corpus(rows, nnz, dim, zipf, g):
    """(indptr int64, cols int32, vals float32) on the device: about nnz distinct sorted columns per row."""
    n = rows * nnz
    u = torch.rand(n, device="cuda", generator=g, dtype=torch.float64)
    if zipf:
        cols = (u.clamp_min(1e-300).pow(-10.0) - 1).clamp_max(2.0 ** 62).to(torch.int64) % dim   # Pareto(0.1)
    else:
        cols = (u * dim).to(torch.int64).clamp_max(dim - 1)
    del u
    key = torch.arange(rows, device="cuda", dtype=torch.int64).repeat_interleave(nnz) * dim + cols
    del cols
    key = torch.unique(key)                                   # sorted: rows in order, columns ascending in a row
    counts = torch.bincount(key // dim, minlength=rows)
    indptr = torch.zeros(rows + 1, dtype=torch.int64, device="cuda")
    indptr[1:] = torch.cumsum(counts, 0)
    cols = (key % dim).to(torch.int32)
    del key
    vals = torch.randint(1, 50, (len(cols),), device="cuda", generator=g).float()
    return indptr, cols, vals


def csr_kernel(h, indptr, cols, vlog, out, st, flags):
    nv.check(nv.load().dsk_wmh_minhash_csr(h, indptr.data_ptr(), cols.data_ptr(), vlog.data_ptr(), len(indptr) - 1,
                                           out.data_ptr(), st.data_ptr(), flags | WMH_INPUT_LOG,
                                           torch.cuda.current_stream().cuda_stream))


def dense_kernel(h, vlog_dense, out, st, flags):
    nv.check(nv.load().dsk_wmh_minhash(h, vlog_dense.data_ptr(), vlog_dense.shape[0], out.data_ptr(), st.data_ptr(),
                                       flags | WMH_INPUT_LOG, torch.cuda.current_stream().cuda_stream))


def event_ms(fn, repeats):
    fn()                                                      # warm-up
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return [round(x, 3) for x in ms]


def densify(indptr, cols, vlog, rows, dim):
    """The given rows as a dense [len(rows), dim] float32 ln(weight) matrix, -inf where the weight is zero."""
    D = torch.full((len(rows), dim), float("-inf"), device="cuda")
    for j, r in enumerate(rows.tolist()):
        a, b = int(indptr[r]), int(indptr[r + 1])
        D[j, cols[a:b].long()] = vlog[a:b]
    return D


def check_rows(h, indptr, cols, vlog, out, st, dim, rows, flags):
    """Do the CSR kernel's rows equal the dense kernel on the same rows densified?"""
    D = densify(indptr, cols, vlog, rows, dim)
    dout = torch.empty((len(rows), SS, 2), dtype=torch.int64, device="cuda")
    dst = torch.empty(len(rows), dtype=torch.int32, device="cuda")
    dense_kernel(h, D, dout, dst, flags)
    torch.cuda.synchronize()
    r = torch.as_tensor(rows, device="cuda")
    return bool(torch.equal(out[r], dout) and torch.equal(st[r], dst))


def kernel_workload(rec, tag, h, indptr, cols, vals, dim, repeats, g):
    n, nnz = len(indptr) - 1, len(cols)
    vlog = torch.log(vals)
    out = torch.empty((n, SS, 2), dtype=torch.int64, device="cuda")
    st = torch.empty(n, dtype=torch.int32, device="cuda")
    ms = event_ms(lambda: csr_kernel(h, indptr, cols, vlog, out, st, 0), repeats)
    best = min(ms) / 1e3
    gather = nnz * 3 * 4 * SS_PAD
    rows = torch.randint(0, n, (48,), device="cuda", generator=g).cpu()
    rows = torch.cat([rows, torch.tensor([0, n - 1]), torch.argmax(indptr[1:] - indptr[:-1]).cpu().view(1)])
    rec[tag] = {"rows": n, "dim": dim, "nnz": nnz, "nnz_per_row": round(nnz / n, 2),
                "max_row_nnz": int((indptr[1:] - indptr[:-1]).max()), "kernel_ms": ms,
                "rows_per_s": round(n / best), "gather_bytes": gather,
                "gather_bytes_per_s": round(gather / best), "gather_share_of_3_35_TBps": round(gather / best / HBM_BYTES_PER_S, 3),
                "evaluations_per_s": round(nnz * SS / best),
                "hbm_bound_ms_if_no_l2_reuse": round(gather / HBM_BYTES_PER_S * 1e3, 2),
                "equals_dense_kernel": check_rows(h, indptr, cols, vlog, out, st, dim, rows, 0)}
    ms_many = event_ms(lambda: csr_kernel(h, indptr, cols, vlog, out, st, WMH_MANY), repeats)
    rec[tag]["kernel_many_ms"] = ms_many
    rec[tag]["many_equals_dense_kernel"] = check_rows(h, indptr, cols, vlog, out, st, dim, rows, WMH_MANY)
    del out, st, vlog
    torch.cuda.empty_cache()


def to_scipy(indptr, cols, vals, dim):
    return sp.csr_matrix((vals.cpu().numpy(), cols.cpu().numpy(), indptr.cpu().numpy()), shape=(len(indptr) - 1, dim))


def wall(fn, repeats):
    out, ts = None, []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(round((time.perf_counter() - t0) * 1e3, 1))
    return out, ts


def old_minhash_many(gen, X):
    """The sparse minhash_many before the CSR kernel: rows densified in 256 MB slabs, the dense kernel on each slab."""
    n = X.shape[0]
    ret = [None] * n
    slab = max(1, (256 << 20) // (4 * gen.dim))
    for r0 in range(0, n, slab):
        dense = np.asarray(X[r0:r0 + slab].toarray(), dtype=np.float32)
        out, status = gen._sample(dense, 0, many=True)
        for i in range(out.shape[0]):
            if status[i] != 1:
                ret[r0 + i] = out[i]
    return ret


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--nnz", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_wmh_sparse.jsonl"))
    a = ap.parse_args()
    # the parameters that shape the measurement; where the line is written is not one of them
    command = "python tools/bench_wmh_sparse.py --rows %d --nnz %d --repeats %d" % (a.rows, a.nnz, a.repeats)
    rec = {"bench": "wmh_sparse", "command": command, "sample_size": SS}
    rec.update(gpu_card())
    g = torch.Generator(device="cuda").manual_seed(0)
    dim = 1 << 20
    t0 = time.perf_counter()
    gen = dsk.WeightedMinHashGenerator(dim, SS, 1)
    h = gen._handle(0)
    rec["generator_setup_s"] = round(time.perf_counter() - t0, 1)

    # (a) Zipf-like columns, end to end as well; (d) and (e) reuse its rows
    indptr, cols, vals = corpus(a.rows, a.nnz, dim, True, g)
    kernel_workload(rec, "a_zipf", h, indptr, cols, vals, dim, a.repeats, g)
    X = to_scipy(indptr, cols, vals, dim)
    sig, rec["a_zipf"]["minhash_batch_scipy_ms"] = wall(lambda: gen.minhash_batch(X), 2)
    rows = np.random.RandomState(0).choice(X.shape[0], 32, replace=False)
    rec["a_zipf"]["minhash_batch_equals_dense"] = bool(np.array_equal(sig[rows], gen.minhash_batch(X[rows].toarray())))
    del sig

    # (d) the old sparse minhash_many on 1,024 rows, per row, against the new one
    Xd = X[:1024]
    old, t_old = wall(lambda: old_minhash_many(gen, Xd), 2)
    new, t_new = wall(lambda: gen.minhash_many(Xd), 2)
    rec["d_minhash_many_1024"] = {"old_densified_ms_per_row": round(min(t_old) / 1024, 3),
                                  "csr_ms_per_row": round(min(t_new) / 1024, 4),
                                  "old_ms": t_old, "csr_ms": t_new,
                                  "equal": all((p is None and q is None) or np.array_equal(p, q.hashvalues)
                                               for p, q in zip(old, new))}

    # (e) one row of 10^6 entries among (a)'s rows
    long_cols = torch.randperm(dim, device="cuda", generator=g)[:1_000_000].sort().values.to(torch.int32)
    long_vals = torch.randint(1, 50, (len(long_cols),), device="cuda", generator=g).float()
    mid = a.rows // 2
    e_indptr = torch.cat([indptr[:mid + 1], indptr[mid:] + len(long_cols)])
    e_cols = torch.cat([cols[:int(indptr[mid])], long_cols, cols[int(indptr[mid]):]])
    e_vals = torch.cat([vals[:int(indptr[mid])], long_vals, vals[int(indptr[mid]):]])
    del X, Xd, old, new
    kernel_workload(rec, "e_long_row", h, e_indptr, e_cols, e_vals, dim, a.repeats, g)
    del e_indptr, e_cols, e_vals, indptr, cols, vals
    torch.cuda.empty_cache()

    # (b) uniform columns
    indptr, cols, vals = corpus(a.rows, a.nnz, dim, False, g)
    kernel_workload(rec, "b_uniform", h, indptr, cols, vals, dim, a.repeats, g)
    del indptr, cols, vals, gen
    torch.cuda.empty_cache()

    # (c) dim 4096, 50 % dense: CSR kernel against the dense kernel, and end to end
    dim_c, n_c = 4096, 100_000
    gen_c = dsk.WeightedMinHashGenerator(dim_c, SS, 1)
    hc = gen_c._handle(0)
    W = torch.randint(1, 50, (n_c, dim_c), device="cuda", generator=g).float()
    W *= torch.rand((n_c, dim_c), device="cuda", generator=g) < 0.5
    Wl = torch.log(W)
    nz = W != 0
    indptr = torch.zeros(n_c + 1, dtype=torch.int64, device="cuda")
    indptr[1:] = torch.cumsum(nz.sum(1), 0)
    cols = nz.nonzero()[:, 1].to(torch.int32)
    vals = W[nz]
    kernel_workload(rec, "c_dense_ish", hc, indptr, cols, vals, dim_c, a.repeats, g)
    dout = torch.empty((n_c, SS, 2), dtype=torch.int64, device="cuda")
    dst = torch.empty(n_c, dtype=torch.int32, device="cuda")
    rec["c_dense_ish"]["dense_kernel_ms"] = event_ms(lambda: dense_kernel(hc, Wl, dout, dst, 0), a.repeats)
    cout = torch.empty_like(dout)
    cst = torch.empty_like(dst)
    csr_kernel(hc, indptr, cols, torch.log(vals), cout, cst, 0)
    rec["c_dense_ish"]["all_rows_equal_dense_kernel"] = bool(torch.equal(cout, dout) and torch.equal(cst, dst))
    Xc = to_scipy(indptr, cols, vals, dim_c)
    del W, Wl, nz, dout, dst, cout, cst
    torch.cuda.empty_cache()
    s1, rec["c_dense_ish"]["minhash_batch_scipy_ms"] = wall(lambda: gen_c.minhash_batch(Xc), 2)
    s2, rec["c_dense_ish"]["minhash_batch_toarray_ms"] = wall(lambda: gen_c.minhash_batch(Xc.toarray()), 2)
    rec["c_dense_ish"]["end_to_end_equal"] = bool(np.array_equal(s1, s2))

    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
