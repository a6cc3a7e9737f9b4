"""Raw text to MinHash signatures (dsk_shingle_count / dsk_shingle_hash + the signature kernel, DESIGN.md section 4m).

    python tools/bench_shingle.py [--docs 1000000] [--repeats 5] [--host-docs 20000] [--out profiles/h100_shingle.jsonl]

Corpus (seeded): --docs documents of 150-300 words drawn from a 50,000-word vocabulary with Zipf-like frequencies
(a Pareto(0.2) draw of the rank: P(rank > r) ~ r^-0.2); about 5 % of the words carry a non-ASCII character (é, ß, ü, 中, rarely an emoji), 5 % of the separators
are newlines.  For word n = 1, word n = 5 and char n = 5, each with sha1_hash32 and xxh32_hash32:
  a  device-resident text (uint8 tensor + int64 offsets) to the [N, 128] signature matrix on the device, through
     shingle.signatures(to_host=False), host clock around the call and a synchronise; and its three stages alone with
     CUDA events: dsk_shingle_count (segmentation, UTF-8 check, counts), dsk_shingle_hash (per-shingle hashing), the
     signature kernel on the resulting tokens
  b  bulk_signatures_device alone on the same tokens, pre-hashed: the signature-only floor
  c  a Python list of str to the host uint64 matrix through shingle.signatures, end to end (encoding, copies included)
  d  the host loop MinHash.bulk([shingles(t, n, unit) for t in texts]) on the first --host-docs documents, per document
Timings are after a warm-up call, --repeats times (c: 3, d: once), reported as min / median / max.  A seeded sample of 1,000
rows of a, b and c (and 1,000 of the host sample for d) is compared with MinHash.bulk over shingles() of those documents.
Prints one JSON line per run and appends it to --out, with the card's name and power limit read in the same process.
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
from datasketch_b200 import _native as nv  # noqa: E402
from datasketch_b200.hashfunc import sha1_hash32, xxh32_hash32  # noqa: E402
from datasketch_b200.minhash import _make_permutations  # noqa: E402
from datasketch_b200.shingle import UNITS, shingles, signatures  # noqa: E402

K = 128
CONFIGS = [("word", 1), ("word", 5), ("char", 5)]
HASHES = [("sha1_hash32", sha1_hash32, 0), ("xxh32_hash32", xxh32_hash32, 1)]


def gpu_card():
    import subprocess
    line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                           "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    name, watts, mhz = [s.strip() for s in line.split(",")]
    return {"gpu": name, "power_limit_w": float(watts), "sm_clock_max_mhz": float(mhz)}


def corpus(n_docs, seed=0):
    """(text uint8, offsets int64) of the synthetic corpus, built in chunks of 20k documents."""
    rs = np.random.RandomState(seed)
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    extra = ["é", "ß", "ü", "中", "\U0001F600"]
    vocab = []
    for i in range(50_000):
        w = bytes(letters[rs.randint(0, 26, rs.randint(2, 11))])
        if rs.rand() < 0.05:
            x = extra[min(int(rs.exponential(1.0)), 4)]
            p = rs.randint(0, len(w) + 1)
            w = w[:p] + x.encode() + w[p:]
        vocab.append(w + b" ")
    wl = np.array([len(w) for w in vocab], dtype=np.int64)
    wstart = np.zeros(len(vocab), dtype=np.int64)
    np.cumsum(wl[:-1], out=wstart[1:])
    flat = np.frombuffer(b"".join(vocab), dtype=np.uint8)
    texts, offs, pos = [], [np.zeros(1, dtype=np.int64)], 0
    for c0 in range(0, n_docs, 20_000):
        nd = min(20_000, n_docs - c0)
        nw = rs.randint(150, 301, nd)
        ids = np.minimum(rs.random_sample(int(nw.sum())) ** -5.0, len(vocab)).astype(np.int64) - 1   # Pareto tail
        lens = wl[ids]
        ends = np.cumsum(lens)
        idx = np.repeat(wstart[ids] - (ends - lens), lens) + np.arange(int(ends[-1]), dtype=np.int64)
        chunk = flat[idx]
        nl = ends[rs.rand(len(ends)) < 0.05] - 1
        chunk[nl] = 0x0A
        doc_end = ends[np.cumsum(nw) - 1]
        texts.append(chunk)
        offs.append(pos + doc_end)
        pos += int(ends[-1])
    return np.concatenate(texts), np.concatenate(offs)


def spread(xs):
    xs = sorted(xs)
    return {"min": round(xs[0], 3), "median": round(xs[len(xs) // 2], 3), "max": round(xs[-1], 3)}


def event_ms(fn, repeats):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return spread(out)


def wall_ms(fn, repeats):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return spread(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-docs", type=int, default=20_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_shingle.jsonl"))
    a = ap.parse_args()
    t0 = time.time()
    text, off = corpus(a.docs)
    gen_s = time.time() - t0
    n = len(off) - 1
    d_text, d_off = torch.from_numpy(text).cuda(), torch.from_numpy(off).cuda()
    texts = [text[off[i]:off[i + 1]].tobytes().decode("utf-8") for i in range(n)]
    perms = _make_permutations(K, 1)
    lib = nv.load()
    rs = np.random.RandomState(1)
    sample = np.sort(rs.choice(n, min(1000, n), replace=False))
    host_n = min(a.host_docs, n)
    host_sample = np.sort(rs.choice(host_n, min(1000, host_n), replace=False))
    rec = {"bench": "shingle", "cmd": " ".join(sys.argv), **gpu_card(), "docs": n, "text_bytes": int(len(text)),
           "num_perm": K, "corpus_seconds": round(gen_s, 1), "runs": []}
    st = torch.cuda.current_stream().cuda_stream
    for unit, nn in CONFIGS:
        for hname, hf, kind in HASHES:
            r = {"unit": unit, "n": nn, "hashfunc": hname}
            # the stages alone, on the C-ABI (the workspace and buffers allocated once)
            wsb = int(lib.dsk_shingle_workspace_size(n, len(text)))
            ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
            tok_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
            status = torch.empty(n + 1, dtype=torch.int32, device="cuda")

            def count():
                nv.check(lib.dsk_shingle_count(d_text.data_ptr(), d_off.data_ptr(), n, len(text), UNITS[unit], nn,
                                               tok_off.data_ptr(), status.data_ptr(), ws.data_ptr(), wsb, st))
            r["a_count_ms"] = event_ms(count, a.repeats)
            total = int(tok_off[n])
            assert int(status[n]) == 0
            tokens = torch.empty(max(total, 4), dtype=torch.int32, device="cuda")

            def hash_():
                nv.check(lib.dsk_shingle_hash(d_text.data_ptr(), d_off.data_ptr(), n, len(text), UNITS[unit], nn, kind, 0,
                                              tok_off.data_ptr(), tokens.data_ptr(), ws.data_ptr(), wsb, st))
            r["a_hash_ms"] = event_ms(hash_, a.repeats)
            r["shingles"] = total
            sig_out = torch.empty((n, K), dtype=torch.int32, device="cuda")
            r["b_sign_ms"] = event_ms(lambda: dsk.engine.bulk_signatures_device(tokens, tok_off, total, perms, d_out=sig_out),
                                      a.repeats)
            b_rows = sig_out[torch.from_numpy(sample).cuda()].cpu().numpy().view(np.uint32).astype(np.uint64)
            del ws
            holder = {}

            def dev_path():
                holder["sig"] = signatures((d_text, d_off), nn, unit, hashfunc=hf, to_host=False)
            r["a_device_text_to_sig_ms"] = wall_ms(dev_path, a.repeats)
            a_rows = holder.pop("sig")[torch.from_numpy(sample).cuda()].cpu().numpy().view(np.uint32).astype(np.uint64)
            del tokens, sig_out
            c_times = []
            for _ in range(3):
                t = time.perf_counter()
                c_sig = signatures(texts, nn, unit, hashfunc=hf)
                c_times.append((time.perf_counter() - t) * 1e3)
            r["c_str_list_to_host_sig_ms"] = spread(c_times)
            c_rows = c_sig[sample]
            del c_sig
            t = time.perf_counter()
            d_sig = np.stack([m.hashvalues for m in dsk.MinHash.bulk([shingles(x, nn, unit) for x in texts[:host_n]],
                                                                      hashfunc=hf)])
            r["d_host_loop_us_per_doc"] = round((time.perf_counter() - t) * 1e6 / host_n, 2)
            want = np.stack([m.hashvalues for m in dsk.MinHash.bulk([shingles(texts[i], nn, unit) for i in sample],
                                                                     hashfunc=hf)])
            want_d = np.stack([m.hashvalues for m in dsk.MinHash.bulk([shingles(texts[i], nn, unit) for i in host_sample],
                                                                       hashfunc=hf)])
            r["sample_rows_equal"] = {"a": bool(np.array_equal(a_rows, want)), "b": bool(np.array_equal(b_rows, want)),
                                      "c": bool(np.array_equal(c_rows, want)),
                                      "d": bool(np.array_equal(d_sig[host_sample], want_d))}
            rec["runs"].append(r)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
