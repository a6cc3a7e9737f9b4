"""The LSHBloom tables bit for bit (SURVEY.md section 8 f3).

``test_lsh_bloom.py`` checks the device Bloom tables statistically: no false negatives, a false-positive rate within the
bound.  Here a short numpy model of the tables fixes every bit.  The band key is the reference's
``x = sum(band) % (2^61 - 1)`` (datasketch/lsh_bloom.py:105); the probe scheme is this library's own (the reference
delegates its tables to pybloomfilter): ``h1 = fmix64(x ^ 0x9E3779B97F4A7C15)``, ``h2 = fmix64(x + 0xD6E8FEB86659FD93) | 1``
and probe q sets bit ``(h1 + q h2) mod 2^64 mod n_bits`` of the band's table, bit ``p & 31`` of word ``p >> 5``.  Saved
``*.bf`` files hold these words, so the scheme must not drift.

CPU part: the C-ABI on the emulated library (2 SMs, so a few hundred documents already run the grid-stride loops).
GPU part: the same sweep with more documents than one grid covers, the single-object API, persistence, and a table
with probe positions above 2^32."""
import shutil
import warnings

import numpy as np
import pytest

from oracle import oracle_np as o

P61 = np.uint64((1 << 61) - 1)
U64 = np.uint64


# ---- the model -----------------------------------------------------------------------------------------------------
def _fmix64(h):
    h = h ^ (h >> U64(33))
    h = h * U64(0xFF51AFD7ED558CCD)
    h = h ^ (h >> U64(33))
    h = h * U64(0xC4CEB9FE1A85EC53)
    return h ^ (h >> U64(33))


def model_keys(sig, b, r):
    """[n, b] uint64 band keys: sum of the band's r values (cannot wrap: r < 2^32) mod 2^61 - 1."""
    s = np.asarray(sig)[:, :b * r].reshape(len(sig), b, r)
    return s.sum(axis=2, dtype=np.uint64) % P61         # summed in uint64 without a uint64 copy of the matrix


def model_positions(sig, b, r, n_bits, n_hashes):
    """[n, b, n_hashes] uint64 bit positions of every probe."""
    x = model_keys(sig, b, r)
    with np.errstate(over="ignore"):
        h1 = _fmix64(x ^ U64(0x9E3779B97F4A7C15))
        h2 = _fmix64(x + U64(0xD6E8FEB86659FD93)) | U64(1)
        q = np.arange(n_hashes, dtype=np.uint64)
        return (h1[..., None] + q * h2[..., None]) % U64(n_bits)


def model_insert(tables, sig, b, r, n_bits, n_hashes):
    pos = model_positions(sig, b, r, n_bits, n_hashes)
    for j in range(b):
        p = pos[:, j].ravel()
        np.bitwise_or.at(tables[j], (p >> U64(5)).astype(np.int64), np.left_shift(np.uint32(1), (p & U64(31)).astype(np.uint32)))


def model_query(tables, sig, b, r, n_bits, n_hashes):
    """bool per row: some band has every probe bit set."""
    pos = model_positions(sig, b, r, n_bits, n_hashes)
    hit = np.zeros(len(sig), dtype=bool)
    for j in range(b):
        p = pos[:, j]
        bit = (tables[j][(p >> U64(5)).astype(np.int64)] >> (p & U64(31)).astype(np.uint32)) & np.uint32(1)
        hit |= bit.astype(bool).all(axis=1)
    return hit


def _words(n_bits):
    return (n_bits + 31) // 32


def _padding_clear(tables, n_bits):
    """The bits past n_bits in the last word of every table are 0."""
    tail = n_bits % 32
    return tail == 0 or not (tables[:, -1] >> np.uint32(tail)).any()


def _random_sig(rs, n, k, hi=1 << 32):
    return rs.randint(0, hi, size=(n, k), dtype=np.uint64).astype(np.uint32)


# (K, b, r, n_bits, n_hashes): bands past lane 31, one probe and 64 probes, the saturated 64-bit minimum table, n_bits
# not a multiple of 32, K not a multiple of 4, b*r < K, K = 4096 (fewer warps per CTA), and rows too long for a warp's
# shared-memory slice: K = 60000 with (2, 10) and K = b*r = 65536
CONFIGS = [
    (128, 9, 13, 20011, 7),
    (66, 33, 2, 1000, 3),
    (128, 64, 2, 64, 1),
    (30, 2, 15, 333, 64),
    (4096, 4, 1000, 5003, 5),
    (60000, 2, 10, 4093, 4),
    (65536, 64, 1024, 2048, 2),
]


def _cfg_id(c):
    return "K%d_b%d_r%d_bits%d_h%d" % c


# ---- CPU: the emulated library ---------------------------------------------------------------------------------------
def _emu_insert(lib, sig, b, r, tables, n_bits, n_hashes):
    sig = np.ascontiguousarray(sig)
    return lib.dsk_bloom_insert(sig.ctypes.data, len(sig), sig.shape[1], b, r, tables.ctypes.data, tables.shape[1],
                                n_bits, n_hashes, None)


def _emu_query(lib, sig, b, r, tables, n_bits, n_hashes):
    sig = np.ascontiguousarray(sig)
    hit = np.full(len(sig), 7, dtype=np.uint8)
    assert lib.dsk_bloom_query(sig.ctypes.data, len(sig), sig.shape[1], b, r, tables.ctypes.data, tables.shape[1],
                               n_bits, n_hashes, hit.ctypes.data, None) == 0
    assert set(np.unique(hit).tolist()) <= {0, 1}
    return hit.astype(bool)


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_emulated_tables_equal_the_model(emu_lib, cfg):
    lib = emu_lib
    k, b, r, n_bits, n_hashes = cfg
    rs = np.random.RandomState(k + b)
    n = 300 if k <= 4096 else 24                      # 300 > 128 documents per emulated grid sweep
    ins = _random_sig(rs, n, k)
    ins[n // 2:n // 2 + 10] = ins[:10]                # duplicate rows
    fresh = _random_sig(rs, n, k)
    fresh[:5] = ins[-5:]                              # inserted rows among the fresh ones
    fresh[5, :r] = ins[n // 3, :r]                    # band 0 alone matches
    fresh[6, (b - 1) * r:b * r] = ins[n // 3 + 1, (b - 1) * r:b * r]   # the last band alone matches
    want = np.zeros((b, _words(n_bits)), dtype=np.uint32)
    model_insert(want, ins, b, r, n_bits, n_hashes)
    got = np.zeros_like(want)
    assert _emu_insert(lib, ins, b, r, got, n_bits, n_hashes) == 0
    assert np.array_equal(got, want)
    assert _padding_clear(got, n_bits)
    q = np.concatenate([ins, fresh])
    hit = _emu_query(lib, q, b, r, got, n_bits, n_hashes)
    assert np.array_equal(hit, model_query(want, q, b, r, n_bits, n_hashes))
    assert hit[:n].all() and hit[n:n + 7].all()        # no false negatives; single-band matches are hits
    if b * r < k:                                     # the columns past b*r are never read
        ins2, q2 = ins.copy(), q.copy()
        ins2[:, b * r:] = _random_sig(rs, n, k - b * r)
        q2[:, b * r:] = _random_sig(rs, len(q), k - b * r)
        got2 = np.zeros_like(want)
        assert _emu_insert(lib, ins2, b, r, got2, n_bits, n_hashes) == 0
        assert np.array_equal(got2, want)
        assert np.array_equal(_emu_query(lib, q2, b, r, got2, n_bits, n_hashes), hit)
    # batches with duplicate rows: the tables of one insert of the union
    parts = np.array_split(np.concatenate([ins, ins[::3]]), 3)
    got3 = np.zeros_like(want)
    for p in parts:
        assert _emu_insert(lib, p, b, r, got3, n_bits, n_hashes) == 0
    assert np.array_equal(got3, want)


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_emulated_band_sums_past_one_grid_sweep(emu_lib):
    lib = emu_lib
    rs = np.random.RandomState(8)
    b, r, k = 9, 13, 128
    n = 2 * 16 * 256 // b + 500                       # n*b > one emulated sweep (2 SMs x 16 CTAs x 256 threads)
    sig = _random_sig(rs, n, k)
    sig[0] = 0xFFFFFFFF
    keys = np.zeros((n, b), dtype=np.uint64)
    assert lib.dsk_band_sums(sig.ctypes.data, n, k, b, r, keys.ctypes.data, None) == 0
    assert np.array_equal(keys, model_keys(sig, b, r))
    assert all(np.array_equal(keys[i], o.bloom_band_keys(sig[i].astype(np.uint64), b, r)) for i in range(0, n, 37))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_emulated_tables_on_the_reference_fixture(emu_lib, golden):
    lib = emu_lib
    sig = np.ascontiguousarray(golden("lsh")["sig"])
    g = golden("bloom")
    b, r = (int(x) for x in g["b_r"])
    n_ins = len(g["keys_inserted"])
    assert np.array_equal(model_keys(sig[:n_ins], b, r), g["keys_inserted"])
    n_bits, n_hashes = 20011, 7
    got = np.zeros((b, _words(n_bits)), dtype=np.uint32)
    assert _emu_insert(lib, sig[:n_ins], b, r, got, n_bits, n_hashes) == 0
    want = np.zeros_like(got)
    model_insert(want, sig[:n_ins], b, r, n_bits, n_hashes)
    assert np.array_equal(got, want)
    hit = _emu_query(lib, sig, b, r, got, n_bits, n_hashes)
    assert np.array_equal(hit, model_query(want, sig, b, r, n_bits, n_hashes))
    assert hit[g["query_all"]].all()


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


def _gpu_insert(d_sig, b, r, d_bits, n_bits, n_hashes):
    import torch
    from datasketch_b200 import _native as nv
    nv.check(nv.load().dsk_bloom_insert(d_sig.data_ptr(), d_sig.shape[0], d_sig.shape[1], b, r, d_bits.data_ptr(),
                                        d_bits.shape[1], n_bits, n_hashes, torch.cuda.current_stream().cuda_stream))


def _gpu_query(d_sig, b, r, d_bits, n_bits, n_hashes):
    import torch
    from datasketch_b200 import _native as nv
    hit = torch.full((d_sig.shape[0],), 7, dtype=torch.uint8, device=d_sig.device)
    nv.check(nv.load().dsk_bloom_query(d_sig.data_ptr(), d_sig.shape[0], d_sig.shape[1], b, r, d_bits.data_ptr(),
                                       d_bits.shape[1], n_bits, n_hashes, hit.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    h = hit.cpu().numpy()
    assert set(np.unique(h).tolist()) <= {0, 1}
    return h.astype(bool)


def _host_bits(d_bits):
    return d_bits.cpu().numpy().view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_device_tables_equal_the_model(cfg):
    import torch
    k, b, r, n_bits, n_hashes = cfg
    rs = np.random.RandomState(k * 3 + b)
    sweep = _sms() * 8 * 8                            # documents per grid: SMs x 8 CTAs x 8 warps
    n = 3 * sweep + 11 if k <= 4096 else 300
    ins = _random_sig(rs, n, k)
    ins[n // 2:n // 2 + 50] = ins[:50]
    fresh = _random_sig(rs, n, k)
    fresh[:5] = ins[-5:]
    fresh[5, :r] = ins[n // 3, :r]
    fresh[6, (b - 1) * r:b * r] = ins[n // 3 + 1, (b - 1) * r:b * r]
    want = np.zeros((b, _words(n_bits)), dtype=np.uint32)
    model_insert(want, ins, b, r, n_bits, n_hashes)
    d_bits = torch.zeros((b, _words(n_bits)), dtype=torch.int32, device="cuda")
    _gpu_insert(_dev(ins), b, r, d_bits, n_bits, n_hashes)
    got = _host_bits(d_bits)
    assert np.array_equal(got, want)
    assert _padding_clear(got, n_bits)
    q = np.concatenate([ins, fresh])
    hit = _gpu_query(_dev(q), b, r, d_bits, n_bits, n_hashes)
    assert np.array_equal(hit, model_query(want, q, b, r, n_bits, n_hashes))
    assert hit[:n].all() and hit[n:n + 7].all()
    if b * r < k:
        ins2, q2 = ins.copy(), q.copy()
        ins2[:, b * r:] = _random_sig(rs, n, k - b * r)
        q2[:, b * r:] = _random_sig(rs, len(q), k - b * r)
        d2 = torch.zeros_like(d_bits)
        _gpu_insert(_dev(ins2), b, r, d2, n_bits, n_hashes)
        assert torch.equal(d2, d_bits)
        assert np.array_equal(_gpu_query(_dev(q2), b, r, d2, n_bits, n_hashes), hit)
    d3 = torch.zeros_like(d_bits)
    for p in np.array_split(np.concatenate([ins, ins[::3], ins[:7]]), 4):
        _gpu_insert(_dev(p), b, r, d3, n_bits, n_hashes)
    assert torch.equal(d3, d_bits)


@pytest.mark.gpu
def test_device_band_sums_past_one_grid_sweep():
    import datasketch_b200 as dsk
    rs = np.random.RandomState(9)
    for k, b, r in ((128, 9, 13), (66, 33, 2)):
        n = 3 * _sms() * 16 * 256 // b + 17           # n*b over three sweeps of SMs x 16 CTAs x 256 threads
        sig = _random_sig(rs, n, k)
        sig[0] = 0xFFFFFFFF
        got = dsk.codec.band_sums(sig, b, r).cpu().numpy().view(np.uint64)
        assert np.array_equal(got, model_keys(sig, b, r)), (k, b, r)
        for i in list(range(0, n, 97)) + [n - 1]:
            assert np.array_equal(got[i], o.bloom_band_keys(sig[i].astype(np.uint64), b, r)), (k, b, r, i)


def _bloom(**kw):
    import datasketch_b200 as dsk
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return dsk.MinHashLSHBloom(**kw)


@pytest.mark.gpu
def test_single_object_api_writes_the_batch_bits(golden):
    import datasketch_b200 as dsk
    sig = golden("lsh")["sig"]
    g = golden("bloom")
    n_ins = len(g["keys_inserted"])
    batch = _bloom(threshold=0.8, num_perm=128, n=1000, fp=0.001)
    b, r = batch.b, batch.r
    assert (b, r) == tuple(int(x) for x in g["b_r"])
    batch.insert_batch(sig[:n_ins])
    want = np.zeros((b, batch.words_per_table), dtype=np.uint32)
    model_insert(want, sig[:n_ins], b, r, batch.n_bits, batch.n_hashes)
    assert np.array_equal(_host_bits(batch._bits), want)
    assert _padding_clear(want, batch.n_bits)
    # one LeanMinHash at a time
    single = _bloom(threshold=0.8, num_perm=128, n=1000, fp=0.001)
    for row in sig[:n_ins]:
        single.insert(dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64)))
    assert np.array_equal(_host_bits(single._bits), want)
    # one band of one document at a time, through the per-band tables
    tables = _bloom(threshold=0.8, num_perm=128, n=1000, fp=0.001)
    for row in sig[:n_ins]:
        for j, (s, e) in enumerate(tables.hashranges):
            tables.hashtables[j].insert(row[s:e])
    assert np.array_equal(_host_bits(tables._bits), want)
    # queries: per object == per batch == the model; no false negatives against the reference's exact answers
    hit = batch.query_batch(sig)
    assert np.array_equal(hit, model_query(want, sig, b, r, batch.n_bits, batch.n_hashes))
    assert hit[g["query_all"]].all()
    for i, row in enumerate(sig):
        assert single.query(dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64))) == bool(hit[i]), i
    for i in range(0, len(sig), 7):
        per_band = [tables.hashtables[j].query(sig[i, s:e]) for j, (s, e) in enumerate(tables.hashranges)]
        assert any(per_band) == bool(hit[i]), i


@pytest.mark.gpu
def test_persistence_keeps_every_bit(tmp_path):
    rs = np.random.RandomState(13)
    n, fp = 5000, 0.01
    bl = _bloom(threshold=0.8, num_perm=128, n=n, fp=fp, save_dir=str(tmp_path / "idx"))
    rows = _random_sig(rs, n, 128)
    bl.insert_batch(rows)
    bl.sync()
    want = _host_bits(bl._bits)
    for i in range(bl.b):
        path = tmp_path / "idx" / ("band-%d.bf" % i)
        assert path.stat().st_size == 32 + 4 * bl.words_per_table
    again = _bloom(threshold=0.8, num_perm=128, n=n, fp=fp, save_dir=str(tmp_path / "idx"))
    assert np.array_equal(_host_bits(again._bits), want)
    q = np.concatenate([rows[:500], _random_sig(rs, 500, 128)])
    assert np.array_equal(again.query_batch(q), bl.query_batch(q))
    for other in (dict(n=n + 1, fp=fp), dict(n=n, fp=0.02)):
        with pytest.raises(ValueError):
            _bloom(threshold=0.8, num_perm=128, save_dir=str(tmp_path / "idx"), **other)


@pytest.mark.gpu
def test_probe_positions_above_two_to_the_32():
    """Tables of 5 * 2^30 bits: a fifth of the probe positions lie above 2^32 (a 32-bit position would wrap)."""
    import torch
    n_bits, b, r, n_hashes, n = 5 << 30, 2, 10, 4, 20_000
    words = _words(n_bits)
    if torch.cuda.mem_get_info()[0] < (4 << 30):
        pytest.skip("needs 4 GB of free device memory")
    rs = np.random.RandomState(21)
    sig = _random_sig(rs, n, b * r)
    pos = model_positions(sig, b, r, n_bits, n_hashes)
    assert 0.15 < (pos >= U64(1 << 32)).mean() < 0.25
    d_bits = torch.zeros((b, words), dtype=torch.int32, device="cuda")   # 2 x 671 MB
    try:
        _gpu_insert(_dev(sig), b, r, d_bits, n_bits, n_hashes)
        for j in range(b):
            p = pos[:, j].ravel()
            w = (p >> U64(5)).astype(np.int64)
            m = np.left_shift(np.uint32(1), (p & U64(31)).astype(np.uint32))
            uw, inv = np.unique(w, return_inverse=True)
            mask = np.zeros(len(uw), dtype=np.uint32)
            np.bitwise_or.at(mask, inv, m)
            d_w = torch.from_numpy(uw).cuda()
            d_m = torch.from_numpy(mask.view(np.int32)).cuda()
            held = d_bits[j, d_w]
            assert torch.equal(held & d_m, d_m), j            # every expected bit is set
            d_bits[j, d_w] = held & ~d_m                       # ... and none other
        assert int(torch.count_nonzero(d_bits)) == 0
        assert _gpu_query(_dev(sig[:100]), b, r, d_bits, n_bits, n_hashes).sum() == 0
    finally:
        del d_bits
        torch.cuda.empty_cache()
