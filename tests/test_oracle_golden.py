"""CPU: pin the oracle (numpy + C restatements) against fixtures produced by the
real reference (oracle/gen_golden.py), incl. the reference's own golden vector."""
import struct

import numpy as np
import pytest

from oracle import oracle_clib as oc
from oracle import oracle_np as o


def test_reference_absolute_golden(golden):
    g = golden("minhash")
    # test/test_minhash.py:109-115 of the reference
    want = [734825475, 960773806, 359816889, 342714745]
    assert g["hello_k4_seed1"].tolist() == want
    hv = o.update_one(o.init_hashvalues(4), o.sha1_hash32(b"Hello"), o.init_permutations(4, 1))
    assert hv.tolist() == want


@pytest.mark.parametrize("k,seed", [(4, 1), (128, 1), (256, 7), (100, 42)])
def test_permutations(golden, k, seed):
    g = golden("minhash")
    p = o.init_permutations(k, seed)
    assert p.dtype == np.uint64 and p.shape == (2, k)
    assert np.array_equal(p, g[f"perm_k{k}_s{seed}"])


def test_c1_bulk(golden):
    g = golden("minhash")
    tok = g["c1_tokens"].reshape(-1)
    off = np.arange(1001, dtype=np.int64) * 64
    P = o.init_permutations(128, 1)
    assert np.array_equal(oc.minhash_bulk_u32tok(tok, off, P), g["c1_sig"])
    sub = o.bulk_signatures_csr(tok[:64 * 50], off[:51], 128, 1)
    assert np.array_equal(sub.astype(np.uint32), g["c1_sig"][:50])


@pytest.mark.parametrize("k", [4, 33, 100, 128, 256])
def test_ragged(golden, k):
    g = golden("minhash")
    tok, off, seed = g[f"rag_k{k}_tokens"], g[f"rag_k{k}_offsets"], int(g[f"rag_k{k}_seed"])
    want = g[f"rag_k{k}_sig"]
    assert np.array_equal(o.bulk_signatures_csr(tok, off, k, seed).astype(np.uint32), want)
    assert np.array_equal(oc.minhash_bulk_u32tok(tok, off, o.init_permutations(k, seed)), want)
    # empty documents keep the all-ones state (minhash.py:167-168, :265-266)
    empties = np.where(np.diff(off) == 0)[0]
    assert len(empties) >= 2 and (want[empties] == 0xFFFFFFFF).all()


def test_long_small_and_u64(golden):
    g = golden("minhash")
    P = o.init_permutations(128, 1)
    assert np.array_equal(oc.minhash_bulk_u32tok(g["long_tokens"], np.array([0, 20000]), P), g["long_sig"])
    assert np.array_equal(oc.minhash_bulk_u32tok(g["small_tokens"], np.array([0, 64]), P), g["small_sig"])
    tok, off = g["u64_tokens"], g["u64_offsets"]
    assert tok.max() >= 2 ** 63
    assert np.array_equal(o.bulk_signatures_csr(tok, off, 64, 3), g["u64_sig"])
    assert np.array_equal(oc.minhash_bulk_u64tok(tok, off, o.init_permutations(64, 3)), g["u64_sig"])


def test_sha1_update_batch(golden):
    g = golden("minhash")
    data = [f"token-{i}".encode() for i in range(1000)]
    hv = o.update_batch(o.init_hashvalues(256), [o.sha1_hash32(x) for x in data], o.init_permutations(256, 7))
    assert np.array_equal(hv, g["sha1_k256_s7_n1000"])
    P = o.init_permutations(128, 7)
    hv = o.update_batch(o.init_hashvalues(128), [o.sha1_hash32(x) for x in data[:500]], P)
    hv = o.update_batch(hv, [o.sha1_hash32(x) for x in data[:700]], P)
    assert np.array_equal(hv, g["sha1_k128_s7_500_700"])


def test_jaccard_merge_union_count(golden):
    g = golden("minhash")
    P = o.init_permutations(128, 1)
    m1 = o.update_batch(o.init_hashvalues(128), range(0, 300), P)
    m2 = o.update_batch(o.init_hashvalues(128), range(150, 450), P)
    assert np.array_equal(m1, g["j_m1"]) and np.array_equal(m2, g["j_m2"])
    assert o.jaccard(m1, m2) == float(g["j_jaccard"])
    assert o.count(m1) == float(g["j_count1"])
    assert np.array_equal(o.merge(m1, m2), g["j_merge"])
    assert np.array_equal(np.minimum.reduce([m1, m2]), g["j_union"])
    sig = np.stack([m1, m2]).astype(np.uint32)
    cnt = oc.jaccard_pairs_u32(sig, np.array([0]), np.array([1]))
    assert cnt[0] / 128.0 == float(g["j_jaccard"])


def test_scalar_bigint_matches_numpy_wrap():
    # the reference arithmetic wraps mod 2^64 BEFORE % p (SURVEY.md section 0 fact 1)
    P = o.init_permutations(16, 3)
    for h in [0, 1, 12, 2 ** 31, 2 ** 32 - 1, 2 ** 40 + 5, 2 ** 64 - 1]:
        hv = o.update_one(o.init_hashvalues(16), h, P)
        want = [min(o.permute_scalar(int(a), int(b), h), 0xFFFFFFFF) for a, b in zip(P[0], P[1])]
        assert hv.tolist() == want


def test_lean_codec(golden):
    g = golden("lean")
    hv, seed = g["hashvalues"], int(g["seed"])
    for bo, nm in {"@": "native", "=": "std", "<": "le", ">": "be", "!": "net"}.items():
        assert o.lean_bytesize(len(hv), bo) == int(g[f"size_{nm}"])
        buf = o.lean_serialize(seed, hv, bo)
        assert np.array_equal(np.frombuffer(buf, np.uint8), g[f"buf_{nm}"])
        s2, hv2 = o.lean_deserialize(buf, bo)
        assert s2 == seed and np.array_equal(hv2, hv)
    # test/test_lean_minhash.py:70-73
    assert o.lean_bytesize(4) == 4 * 4 + 4 + 8
    assert np.array_equal(oc.lean_pack_le(g["batch_sig"], 9), g["batch_recs"])
    assert struct.calcsize("@qi") == 12  # native layout has no padding between q and i


def test_wmh(golden):
    g = golden("wmh")
    for tag in ("small", "tiny"):
        dim, ss, seed = [int(x) for x in g[f"{tag}_cfg"]]
        rs, ln_cs, betas = o.wmh_params(dim, ss, seed)
        assert np.array_equal(rs, g[f"{tag}_rs"]) and np.array_equal(ln_cs, g[f"{tag}_ln_cs"])
        assert np.array_equal(betas, g[f"{tag}_betas"])
        out = np.stack([o.wmh_minhash(v, rs, ln_cs, betas) for v in g[f"{tag}_v"]])
        assert out.dtype == np.int64 and np.array_equal(out, g[f"{tag}_out"])
    dim, ss, seed = [int(x) for x in g["c4_cfg"]]
    rs, ln_cs, betas = o.wmh_params(dim, ss, seed)
    assert np.array_equal(rs[:2, :64], g["c4_rs_head"]) and np.array_equal(betas[:2, :64], g["c4_betas_head"])
    sums = np.array([rs.astype(np.float64).sum(), ln_cs.astype(np.float64).sum(), betas.astype(np.float64).sum()])
    assert np.array_equal(sums, g["c4_sums"])
    out = np.stack([o.wmh_minhash(v, rs, ln_cs, betas) for v in g["c4_v"]])
    assert np.array_equal(out, g["c4_out"])
    with pytest.raises(ValueError):
        o.wmh_minhash(np.zeros(dim), rs, ln_cs, betas)
    with pytest.raises(ValueError):
        o.wmh_minhash(np.ones(3), rs, ln_cs, betas)


def test_lsh_params_keys_query(golden):
    g = golden("lsh")
    for thr, k, w0, w1, b, r in g["params"]:
        if k > 128:
            continue  # K=256 grid search is slow; covered once by the API test
        assert o.lsh_optimal_param(float(thr), int(k), float(w0), float(w1)) == (int(b), int(r))
    b, r = [int(x) for x in g["b_r"]]
    assert (b, r) == (9, 13)
    sig = g["sig"].astype(np.uint64)
    keys0 = o.lsh_band_keys(sig[0], b, r)
    assert all(len(x) == 8 * r for x in keys0)
    assert np.array_equal(np.frombuffer(b"".join(keys0), np.uint8).reshape(b, 8 * r), g["keys_doc0"])
    assert np.array_equal(oc.band_keys_be(g["sig"][:1], b, r)[0], g["keys_doc0"])
    lsh = o.DictLSH(128, b, r)
    for i, row in enumerate(sig):
        lsh.insert(i, row)
    ptr, idx = g["query_ptr"], g["query_idx"]
    for i, row in enumerate(sig):
        assert sorted(lsh.query(row)) == idx[ptr[i]:ptr[i + 1]].tolist()
    with pytest.raises(ValueError):
        lsh.insert(0, sig[0])
    # reference-pinned candidate set (test/test_lsh.py:109-125)
    ab, ar = [int(x) for x in g["abc_b_r"]]
    l2 = o.DictLSH(32, ab, ar)
    for i, row in enumerate(g["abc_sig"]):
        l2.insert(i, row)
    assert sorted(l2.query(g["abc_sig"][0])) == g["abc_query0"].tolist() == [0, 1]


def test_wmh_minhash_many(golden):
    """The oracle's minhash_many restatement against the reference's own outputs (dense == sparse there)."""
    g = golden("wmh_many")
    for tag in ("small", "tiny", "mid"):
        dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
        got = o.wmh_minhash_many(g[f"{tag}_X"], *o.wmh_params(dim, ss, seed))
        null = g[f"{tag}_null"]
        assert [m is None for m in got] == null.tolist() and null.any()
        for i, m in enumerate(got):
            if m is not None:
                assert m.dtype == int and np.array_equal(m, g[f"{tag}_out"][i])
    with pytest.raises(ValueError):
        o.wmh_minhash_many(np.ones(5), *o.wmh_params(5, 4, 1))
    with pytest.raises(ValueError):
        o.wmh_minhash_many(np.ones((2, 3)), *o.wmh_params(5, 4, 1))


def _np_log32(V):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(np.asarray(V, dtype=np.float32))


def test_wmh_from_log(golden):
    """The vectorised float32 step sequence equals the per-vector restatements and the reference's own outputs,
    including the special-weight rows (zeros, -0.0, negative, NaN, +-inf, subnormals, FLT_MAX) of wmh_special."""
    g = golden("wmh")
    for tag in ("small", "tiny", "c4"):
        dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
        out, st = o.wmh_from_log(_np_log32(g[f"{tag}_v"]), *o.wmh_params(dim, ss, seed))
        assert not st.any() and np.array_equal(out, g[f"{tag}_out"])
    g = golden("wmh_many")
    for tag in ("small", "tiny", "mid"):
        dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
        out, st = o.wmh_from_log(_np_log32(g[f"{tag}_X"]), *o.wmh_params(dim, ss, seed), many=True)
        null = g[f"{tag}_null"]
        assert np.array_equal(st == 1, null) and not (st == 2).any()
        assert np.array_equal(out[~null], g[f"{tag}_out"][~null]) and not out[null].any()
    rs = np.random.RandomState(3)
    V = (rs.lognormal(0, 3, (40, 259)) * (rs.rand(40, 259) < 0.6)).astype(np.float32)
    V[:, 7] = 1.0
    par = o.wmh_params(259, 37, 9)
    out, st = o.wmh_from_log(_np_log32(V), *par)
    assert not st.any() and np.array_equal(out, np.stack([o.wmh_minhash(v, *par) for v in V]))
    out, st = o.wmh_from_log(_np_log32(V), *par, many=True)
    assert not st.any() and np.array_equal(out, np.stack(o.wmh_minhash_many(V, *par)))
    g = golden("wmh_special")
    X = g["X"]
    for tag in ("a", "b"):
        dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
        par = o.wmh_params(dim, ss, seed)
        out, st = o.wmh_from_log(_np_log32(X), *par)
        err = g[f"{tag}_err"]
        assert np.array_equal(st == 1, err == "ValueError") and np.array_equal(st == 2, err == "OverflowError")
        ok = err == ""
        assert ok.sum() >= 5 and np.array_equal(out[ok], g[f"{tag}_out"][ok])
        out, st = o.wmh_from_log(_np_log32(X), *par, many=True)
        null = g[f"{tag}_many_null"]
        assert np.array_equal(st == 1, null) and (st == 2).sum() >= 5
        assert np.array_equal(out, g[f"{tag}_many_out"])
        with np.errstate(invalid="ignore"):
            per_row = o.wmh_minhash_many(X, *par)
        assert [m is None for m in per_row] == null.tolist()
        assert all(np.array_equal(m, out[i]) for i, m in enumerate(per_row) if m is not None)


def test_wmh_terms64():
    """The float64 evaluation agrees with the float32 one to a few float32 ulps, and exactly on exact inputs."""
    rs, ln_cs, betas = o.wmh_params(50, 8, 2)
    vlog = _np_log32(np.random.RandomState(0).uniform(0.1, 10, 50))
    for many in (False, True):
        arg, ln_a = o.wmh_terms64(vlog, rs, ln_cs, betas, many)
        arg32 = vlog / rs + betas
        t = np.floor(arg32)
        ln_a32 = ln_cs - (t - betas + 1) * rs if many else ln_cs - (t - betas) * rs - rs
        same_t = np.floor(arg) == t
        scale_arg = np.abs(vlog / rs) + betas                     # float32 rounding is relative to the operands
        scale_ln_a = np.abs(ln_cs) + np.abs(t - betas + 1) * rs + rs
        assert same_t.mean() > 0.99 and np.all(np.abs(arg - arg32) <= 2 * np.spacing(scale_arg))
        assert np.all((np.abs(ln_a - ln_a32) <= 4 * np.spacing(scale_ln_a))[same_t])
    arg, ln_a = o.wmh_terms64(np.float32(3.0), np.float32(2.0), np.float32(0.5), np.float32(0.25))
    assert arg == 1.75 and ln_a == 0.5 - (1.0 - 0.25) * 2.0 - 2.0


def test_token_hashes(golden):
    """xxh32 restatement vs the values the `xxhash` package produced; MurmurHash3 x86_32 vs published vectors
    (SMHasher / mmh3 documentation); the product's single-token host functions agree with both."""
    from datasketch_b200 import hashfunc as hf
    g = golden("hashes")
    blob, off = g["blob"], g["off"]
    toks = [bytes(blob[off[i]:off[i + 1]]) for i in range(len(off) - 1)]
    for seed in (0, 1, 0x9747B28C):
        want = g[f"xxh32_seed{seed}"].tolist()
        assert [o.xxh32(t, seed) for t in toks] == want
        assert [hf.xxh32_hash32(t, seed) for t in toks] == want
    vectors = {(b"", 0): 0, (b"", 1): 0x514E28B7, (b"", 0xFFFFFFFF): 0x81F16F39, (b"\xff\xff\xff\xff", 0): 0x76293B50,
               (b"!Ce\x87", 0): 0xF55B516B, (b"!Ce\x87", 0x5082EDEE): 0x2362F9DE, (b"!Ce", 0): 0x7E4A8634,
               (b"!C", 0): 0xA0F7B07A, (b"!", 0): 0x72661CF4, (b"\0\0\0\0", 0): 0x2362F9DE, (b"aaaa", 0x9747B28C): 0x5A97808A,
               (b"hello", 0): 0x248BFA47, (b"foo", 0): 0xF6A5C420, (b"Hello, world!", 0): 0xC0363E43,
               (b"The quick brown fox jumps over the lazy dog", 0): 0x2E4FF723}
    for (data, seed), want in vectors.items():
        assert o.murmur3_32(data, seed) == want and hf.murmur3_hash32(data, seed) == want, (data, seed)
    rs = np.random.RandomState(5)
    for _ in range(200):
        d = bytes(rs.randint(0, 256, size=rs.randint(0, 70)).astype(np.uint8))
        s32 = int(rs.randint(0, 1 << 32))
        assert hf.murmur3_hash32(d, s32) == o.murmur3_32(d, s32) and hf.xxh32_hash32(d, s32) == o.xxh32(d, s32)
    assert hf.sha1_hash32(b"Hello") == o.sha1_hash32(b"Hello")


def test_bloom_band_keys_and_redis_layout(golden):
    """The oracle's LSHBloom keys and Redis layout against what the reference's own code wrote when it ran on the
    in-memory stand-ins for pybloomfilter / redis (oracle/gen_golden.py: gen_bloom, gen_storage)."""
    import pickle
    sig = golden("lsh")["sig"]
    g = golden("bloom")
    b, r = (int(x) for x in g["b_r"])
    keys = g["keys_inserted"]
    for i in range(len(keys)):
        assert np.array_equal(o.bloom_band_keys(sig[i].astype(np.uint64), b, r), keys[i])
    for thr, k, bb, rr in g["params"]:
        assert o.lsh_optimal_param(float(thr), int(k)) == (int(bb), int(rr))
    # exact-membership tables: a row is a duplicate iff one of its band keys was inserted for that band
    seen = [set(keys[:, j].tolist()) for j in range(b)]
    want = [any(int(x) in seen[j] for j, x in enumerate(o.bloom_band_keys(row.astype(np.uint64), b, r))) for row in sig]
    assert want == g["query_all"].tolist() and all(want[:len(keys)]) and not all(want)
    s = golden("storage")
    for name, mk in (("pickled", lambda i: ("doc", i)), ("bytes", lambda i: b"k%04d" % i)):
        state = pickle.loads(s[name + "_state"].tobytes())
        bb, rr = (int(x) for x in s[name + "_b_r"])
        got = o.redis_layout([mk(i) for i in range(120)], sig[:120].astype(np.uint64), bb, rr, b"gpuidx",
                             prepickle=(name == "pickled"))
        assert got == state
        assert set(state["hash"]) == {b"gpuidx_keys"} | {b"gpuidx_bucket_" + bytes([0, i]) for i in range(bb)}
