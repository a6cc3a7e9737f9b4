"""MinHashLSHBloom.insert_unique against the flows it replaces.

    python tools/bench_bloom_unique.py [--batches 100000 1000000] [--prefill 10000000] [--loop-rows 5000] [--rounds 3]
                                       [--out profiles/h100_bloom_unique.jsonl]

Index: MinHashLSHBloom(threshold=0.8, num_perm=128, n=100_000_000, fp=1e-5), pre-filled with --prefill seeded random rows
through insert_batch.  Each batch is seeded and mixed as DESIGN.md §4e's: 40 % copies of pre-filled rows with 10 % of the
positions resampled, 20 % unrelated rows, 20 % drift chains of 5 rows (5 % resampled per step), 20 % exact copies of
earlier batch rows.  Before timing, once per batch: insert_unique's keep mask must equal the loop's (run over the batch's
probe bits, with the bits set before the call read from the tables) and its tables must equal the prior tables plus
insert_batch of the loop's kept rows.  Then, alternating, --rounds rounds after a warm-up, the tables restored from a
device copy before every call, each call timed with CUDA events up to a synchronised device:
  insert_unique(batch, to_host=False);
  query_batch(batch, to_host=False) + insert_batch(batch[~dup]) (reported with the rows it keeps that the loop drops);
  the row-by-row loop `if not query(m): insert(m)` over the first --loop-rows rows (per row, one round).
Prints one JSON line and appends it to --out, with the card's name and power limit read in the same process.
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import datasketch_b200 as dsk  # noqa: E402
from datasketch_b200 import _native as nv  # noqa: E402
from test_lsh_bloom_exact import model_positions  # noqa: E402
from test_lsh_bloom_unique import loop_on_probe_bits  # noqa: E402


def gpu_card():
    """The card's name, power limit and top SM clock, read in the same process as the timings beside them."""
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def ev(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


def _resample(rs, rows, frac):
    rows = rows.copy()
    mask = rs.random_sample(rows.shape) < frac
    rows[mask] = rs.randint(0, 1 << 32, size=int(mask.sum()), dtype=np.uint64).astype(np.uint32)
    return rows


def make_batch(n, k, prefilled, seed):
    """[n, k] uint32: 40 % perturbed copies of pre-filled rows, 20 % unrelated, 20 % drift chains of 5, 20 % exact
    copies of earlier batch rows (placed after all of them)"""
    rs = np.random.RandomState(seed)
    n_copy, n_new, n_chain = int(0.4 * n), int(0.2 * n), int(0.2 * n) // 5 * 5
    parts = [_resample(rs, prefilled[rs.randint(0, len(prefilled), n_copy)], 0.10),
             rs.randint(0, 1 << 32, size=(n_new, k), dtype=np.uint64).astype(np.uint32)]
    chains = [rs.randint(0, 1 << 32, size=(n_chain // 5, k), dtype=np.uint64).astype(np.uint32)]
    for _ in range(4):
        chains.append(_resample(rs, chains[-1], 0.05))
    parts.append(np.stack(chains, axis=1).reshape(n_chain, k))   # each chain's 5 rows in order
    head = np.concatenate(parts)
    tail = head[rs.randint(0, len(head), n - len(head))]
    return np.ascontiguousarray(np.concatenate([head, tail]))


def loop_keep(bl, batch):
    """the loop's keep mask, from the tables as they are now"""
    pos = model_positions(batch, bl.b, bl.r, bl.n_bits, bl.n_hashes)
    preset = np.empty(pos.shape, dtype=bool)
    band = torch.arange(bl.b, device="cuda").view(1, -1, 1)
    for lo in range(0, len(batch), 100_000):
        p = torch.from_numpy(pos[lo:lo + 100_000].astype(np.int64)).cuda()
        words = bl._bits[band, p >> 5]
        preset[lo:lo + 100_000] = ((words >> (p & 31)) & 1).bool().cpu().numpy()
    return loop_on_probe_bits(pos, preset, bl.n_bits)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--prefill", type=int, default=10_000_000)
    ap.add_argument("--loop-rows", type=int, default=5000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bloom_unique.jsonl"))
    args = ap.parse_args()
    nv.require_device(0)
    k = 128
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        bl = dsk.MinHashLSHBloom(threshold=0.8, num_perm=k, n=100_000_000, fp=1e-5)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    first = None
    for lo in range(0, args.prefill, 1_000_000):
        rows = torch.randint(-(1 << 31), 1 << 31, (min(1_000_000, args.prefill - lo), k), dtype=torch.int32, device="cuda",
                             generator=gen)
        bl.insert_batch(rows)
        if first is None:
            first = rows[:200_000].cpu().numpy().view(np.uint32)
        del rows
    saved = bl._bits.clone()
    torch.cuda.synchronize()
    lib = nv.load()
    res = {"bench": "bloom_unique", "num_perm": k, "b": bl.b, "r": bl.r, "n_bits": bl.n_bits, "n_hashes": bl.n_hashes,
           "prefill": args.prefill, "rounds": args.rounds, "command": " ".join(sys.argv), **gpu_card()}
    for n in args.batches:
        batch = make_batch(n, k, first, seed=n)
        d_batch = torch.from_numpy(batch.view(np.int32)).cuda()
        t0 = time.time()
        want = loop_keep(bl, batch)
        model_s = time.time() - t0
        keep = bl.insert_unique(d_batch, to_host=False).cpu().numpy()
        after = bl._bits.clone()
        bl._bits.copy_(saved)
        bl.insert_batch(d_batch[torch.from_numpy(want).cuda()])
        equal = bool(np.array_equal(keep, want)) and bool(torch.equal(after, bl._bits))
        del after
        if not equal:
            raise SystemExit("insert_unique differs from the loop at n = %d" % n)

        def unique():
            return bl.insert_unique(d_batch, to_host=False)

        def two_step():
            dup = bl.query_batch(d_batch, to_host=False)
            bl.insert_batch(d_batch[~dup])
            return dup

        t_u, t_2 = [], []
        for rnd in range(args.rounds + 1):
            bl._bits.copy_(saved)
            tu, _ = ev(unique)
            bl._bits.copy_(saved)
            t2, dup = ev(two_step)
            if rnd:
                t_u.append(tu)
                t_2.append(t2)
        dup = dup.cpu().numpy()
        extra = int((~dup & ~want).sum())
        # the row-by-row loop through the single-object API, on a slice
        bl._bits.copy_(saved)
        sl = batch[:args.loop_rows]
        objs = [dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)) for row in sl]
        loop_keep_sl = np.zeros(len(sl), dtype=bool)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j, m in enumerate(objs):
            if not bl.query(m):
                bl.insert(m)
                loop_keep_sl[j] = True
        torch.cuda.synchronize()
        loop_ms = (time.perf_counter() - t0) * 1e3
        loop_equal = bool(np.array_equal(loop_keep_sl, want[:len(sl)]))
        bl._bits.copy_(saved)
        ws = int(lib.dsk_bloom_unique_workspace_size(n, k, bl.b, bl.r, bl.n_hashes))
        res["n%d" % n] = {"kept": int(want.sum()), "dropped_by_tables": int(_pre_dropped(bl, d_batch)),
                          "insert_unique_ms": [round(x, 3) for x in t_u],
                          "query_insert_ms": [round(x, 3) for x in t_2], "query_insert_extra_kept": extra,
                          "row_loop_rows": len(sl), "row_loop_us_per_row": round(loop_ms * 1e3 / len(sl), 2),
                          "row_loop_equal": loop_equal, "workspace_bytes": ws, "equal_to_loop": equal,
                          "model_loop_s": round(model_s, 1)}
        print(json.dumps({n: res["n%d" % n]}), flush=True)
        del d_batch
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


def _pre_dropped(bl, d_batch):
    return int(bl.query_batch(d_batch, to_host=False).sum())


if __name__ == "__main__":
    main()
