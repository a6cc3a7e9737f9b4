"""MinHashLSHBloom.insert_unique: the query-then-insert loop over a whole batch on the device (DESIGN.md §4i).

The oracle is the loop itself over the numpy model of ``test_lsh_bloom_exact.py``: for each row in order, ``model_query``
on the row, then ``model_insert`` if it missed.  After every call the keep mask must equal the loop's, every table word
(padding bits included) the loop's tables, and the tables the prior state plus ``insert_batch(sig[keep])``.

CPU part: the C-ABI on the emulated library, and the resolution under ThreadSanitizer.  GPU part: the same cases through
the Python API, with more rows than one grid, probe positions above 2^32 and the class's own row-by-row loop."""
import os
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_lsh_bloom_exact import (CONFIGS, U64, _cfg_id, _padding_clear, _random_sig, _words,  # noqa: E402
                                  model_insert, model_positions, model_query)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
DSK_OK, DSK_ERR_INVALID, DSK_ERR_ALIGN = 0, 1, 4


# ---- the oracle ------------------------------------------------------------------------------------------------------
def model_loop(tables, sig, b, r, n_bits, n_hashes):
    """(keep, tables after) of the loop over the rows of sig, from a copy of `tables`."""
    t = tables.copy()
    keep = np.zeros(len(sig), dtype=bool)
    for j in range(len(sig)):
        row = sig[j:j + 1]
        if not model_query(t, row, b, r, n_bits, n_hashes)[0]:
            model_insert(t, row, b, r, n_bits, n_hashes)
            keep[j] = True
    return keep, t


def loop_on_probe_bits(pos, preset, n_bits):
    """The same loop over the batch's own probe bits: pos [n, b, h] positions, preset [n, b, h] True where the bit was
    set before the call.  Needs no copy of the tables, so it also runs against tables too large for the host."""
    n, b, h = pos.shape
    keys = pos + (np.arange(b, dtype=np.uint64) * U64(n_bits))[None, :, None]
    uniq, ids = np.unique(keys.ravel(), return_inverse=True)
    ids = ids.reshape(n, b, h)
    state = np.zeros(len(uniq), dtype=bool)
    state[ids[preset]] = True
    keep = np.zeros(n, dtype=bool)
    for j in range(n):
        ij = ids[j]
        if state[ij].all(axis=1).any():
            continue
        state[ij] = True
        keep[j] = True
    return keep


def _preset(tables, pos):
    b = pos.shape[1]
    band = np.arange(b)[None, :, None]
    return ((tables[band, (pos >> U64(5)).astype(np.int64)] >> (pos & U64(31)).astype(np.uint32)) & np.uint32(1)).astype(bool)


# ---- the emulated library --------------------------------------------------------------------------------------------
def _emu_unique(lib, sig, b, r, tables, n_bits, n_hashes):
    sig = np.ascontiguousarray(sig, dtype=np.uint32)
    n, k = sig.shape
    need = lib.dsk_bloom_unique_workspace_size(n, k, b, r, n_hashes)
    ws = np.zeros(need // 8 + 2, dtype=np.uint64)      # 16-byte aligned by numpy's allocator
    keep = np.full(n, 7, dtype=np.uint8)
    rc = lib.dsk_bloom_unique(sig.ctypes.data if n else None, n, k, b, r, tables.ctypes.data, tables.shape[1], n_bits,
                              n_hashes, ws.ctypes.data if n else None, need, keep.ctypes.data if n else None, None)
    assert rc == DSK_OK
    assert set(np.unique(keep).tolist()) <= {0, 1}
    return keep.astype(bool)


def _emu_insert(lib, sig, b, r, tables, n_bits, n_hashes):
    sig = np.ascontiguousarray(sig, dtype=np.uint32)
    assert lib.dsk_bloom_insert(sig.ctypes.data, len(sig), sig.shape[1], b, r, tables.ctypes.data, tables.shape[1], n_bits,
                                n_hashes, None) == DSK_OK


def _check_emu(lib, tables, batch, b, r, n_bits, n_hashes):
    """insert_unique of `batch` into `tables` (in place) == the loop; returns keep."""
    before = tables.copy()
    want_keep, want_tables = model_loop(tables, batch, b, r, n_bits, n_hashes)
    keep = _emu_unique(lib, batch, b, r, tables, n_bits, n_hashes)
    assert np.array_equal(keep, want_keep), np.flatnonzero(keep != want_keep)[:20]
    assert np.array_equal(tables, want_tables)
    assert _padding_clear(tables, n_bits)
    again = before.copy()
    if keep.any():
        _emu_insert(lib, batch[keep], b, r, again, n_bits, n_hashes)
    assert np.array_equal(again, tables)
    return keep


def _tables(b, n_bits):
    return np.zeros((b, _words(n_bits)), dtype=np.uint32)


needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


# ---- batch builders --------------------------------------------------------------------------------------------------
def _copies_batch(rs, k, prior, n):
    """fresh rows, exact copies inside the batch (one bucket of hundreds), copies of rows inserted before the call"""
    batch = _random_sig(rs, n, k)
    batch[n // 4:n // 4 + min(300, n // 2)] = batch[n // 5]
    src = rs.randint(0, n - n // 10, size=n // 10)
    batch[n - n // 10:] = batch[src]
    m = min(len(prior), n // 10)
    batch[1:1 + 2 * m:2] = prior[:m]
    return batch


def _drift_chain(rs, n, k, b, r):
    """row j copies exactly one band of row j - 1 (a different band each time) and nothing else: the loop keeps every
    other row, and each row's decision waits for the one before"""
    sig = _random_sig(rs, n, k)
    for j in range(1, n):
        t = j % b
        sig[j, t * r:(t + 1) * r] = sig[j - 1, t * r:(t + 1) * r]
    return sig


# ---- CPU: the emulated library ---------------------------------------------------------------------------------------
@needs_gxx
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_emulated_geometries(emu_lib, cfg):
    k, b, r, n_bits, n_hashes = cfg
    rs = np.random.RandomState(k + 7 * b)
    n = 400 if k <= 4096 else 40
    prior = _random_sig(rs, n // 2, k)
    tables = _tables(b, n_bits)
    _emu_insert(emu_lib, prior, b, r, tables, n_bits, n_hashes)
    batch = _copies_batch(rs, k, prior, n)
    t0 = tables.copy()
    keep = _check_emu(emu_lib, tables, batch, b, r, n_bits, n_hashes)
    assert not keep.all() and (keep.any() or n_bits < 1000)   # the 64-bit tables are saturated by the prior rows
    if b * r < k:   # the columns past b*r are never read
        batch2 = batch.copy()
        batch2[:, b * r:] = _random_sig(rs, n, k - b * r)
        assert np.array_equal(_check_emu(emu_lib, t0, batch2, b, r, n_bits, n_hashes), keep)
        assert np.array_equal(t0, tables)


@needs_gxx
def test_emulated_copies_inside_and_before_the_batch(emu_lib):
    k, b, r, n_bits, n_hashes = 128, 9, 13, 1 << 20, 7
    rs = np.random.RandomState(3)
    prior = _random_sig(rs, 100, k)
    tables = _tables(b, n_bits)
    _emu_insert(emu_lib, prior, b, r, tables, n_bits, n_hashes)
    batch = _random_sig(rs, 700, k)
    batch[100:600] = batch[50]                      # a bucket of 500 exact copies
    batch[20:40] = prior[:20]                       # copies of rows inserted before the call
    keep = _check_emu(emu_lib, tables, batch, b, r, n_bits, n_hashes)
    assert keep[50] and not keep[100:600].any() and not keep[20:40].any()


@needs_gxx
def test_emulated_long_drift_chain(emu_lib):
    k, b, r, n_bits, n_hashes = 32, 4, 8, 1 << 22, 3
    rs = np.random.RandomState(5)
    sig = _drift_chain(rs, 2100, k, b, r)
    keep = _check_emu(emu_lib, _tables(b, n_bits), sig, b, r, n_bits, n_hashes)
    assert keep.tolist() == [j % 2 == 0 for j in range(2100)]


def _coverage_kinds(tables0, batch, keep, b, r, n_bits, n_hashes):
    """Counts over (row, band) of the loop's run: covered only by the union of two or more kept earlier rows; covered by
    pre-set bits plus one kept row (neither alone); covered when the dropped earlier rows' bits are counted too but
    not by the kept ones (a dropped contributor, which must not cover)."""
    pos = model_positions(batch, b, r, n_bits, n_hashes)
    pre = _preset(tables0, pos)
    union = single_pre = dropped = 0
    for j in range(len(batch)):
        for t in range(b):
            mine = set(pos[j, t][~pre[j, t]].tolist())
            if not mine:
                continue
            kept_sets = [set(pos[i, t].tolist()) for i in range(j) if keep[i]]
            all_sets = [set(pos[i, t].tolist()) for i in range(j)]
            by_kept = mine <= set().union(*kept_sets)
            if by_kept and not any(set(pos[j, t].tolist()) <= s for s in kept_sets):
                if any(mine <= s for s in kept_sets):
                    single_pre += 1
                else:
                    union += 1
            if not by_kept and mine <= set().union(*all_sets):
                dropped += 1
    return union, single_pre, dropped


TINY = [(64, 2), (97, 3), (128, 4), (256, 4), (200, 2)]


def _tiny_case(n_bits, n_hashes):
    """(prior rows, batch) for tiny tables with K = 16, (b, r) = (4, 4): the prior rows pre-set some bits"""
    rs = np.random.RandomState(n_bits + n_hashes)
    prior = _random_sig(rs, max(3, n_bits // 40), 16)
    batch = _random_sig(rs, max(60, n_bits // 2), 16)
    batch[30:33] = batch[3]
    return prior, batch


@needs_gxx
@pytest.mark.parametrize("n_bits,n_hashes", TINY)
def test_emulated_union_coverage_in_tiny_tables(emu_lib, n_bits, n_hashes):
    k, b, r = 16, 4, 4
    prior, batch = _tiny_case(n_bits, n_hashes)
    tables = _tables(b, n_bits)
    _emu_insert(emu_lib, prior, b, r, tables, n_bits, n_hashes)
    t0 = tables.copy()
    keep = _check_emu(emu_lib, tables, batch, b, r, n_bits, n_hashes)
    union, single_pre, dropped = _coverage_kinds(t0, batch, keep, b, r, n_bits, n_hashes)
    assert union > 0 and single_pre > 0 and dropped > 0, (union, single_pre, dropped)


@needs_gxx
def test_emulated_repeated_probe_positions(emu_lib):
    k, b, r, n_bits, n_hashes = 30, 2, 15, 100, 64
    rs = np.random.RandomState(11)
    batch = _random_sig(rs, 80, k)
    pos = model_positions(batch, b, r, n_bits, n_hashes)
    repeats = sum(len(set(pos[j, t].tolist())) < n_hashes for j in range(len(batch)) for t in range(b))
    assert repeats > 0
    _check_emu(emu_lib, _tables(b, n_bits), batch, b, r, n_bits, n_hashes)


@needs_gxx
def test_emulated_batches(emu_lib):
    """an empty batch, an all-dropped batch, the same batch twice, and A then B == A ++ B"""
    k, b, r, n_bits, n_hashes = 64, 8, 8, 5003, 3
    rs = np.random.RandomState(17)
    tables = _tables(b, n_bits)
    assert _emu_unique(emu_lib, np.zeros((0, k), dtype=np.uint32), b, r, tables, n_bits, n_hashes).shape == (0,)
    assert not tables.any()
    a = _copies_batch(rs, k, _random_sig(rs, 5, k), 150)
    keep = _check_emu(emu_lib, tables, a, b, r, n_bits, n_hashes)
    assert keep.any()
    assert not _check_emu(emu_lib, tables, a, b, r, n_bits, n_hashes).any()       # the same batch again keeps nothing
    assert not _check_emu(emu_lib, tables, a[keep][::-1].copy(), b, r, n_bits, n_hashes).any()   # all dropped
    bb = _copies_batch(rs, k, a, 120)
    t1, t2 = _tables(b, n_bits), _tables(b, n_bits)
    k1 = np.concatenate([_check_emu(emu_lib, t1, a, b, r, n_bits, n_hashes), _check_emu(emu_lib, t1, bb, b, r, n_bits, n_hashes)])
    k2 = _check_emu(emu_lib, t2, np.concatenate([a, bb]), b, r, n_bits, n_hashes)
    assert np.array_equal(k1, k2) and np.array_equal(t1, t2)


def test_probe_bit_loop_equals_the_loop():
    """loop_on_probe_bits (used for the large cases and the benchmark) == model_loop"""
    rs = np.random.RandomState(23)
    for k, b, r, n_bits, n_hashes in [(16, 4, 4, 64, 2), (128, 9, 13, 20011, 7), (30, 2, 15, 100, 64)]:
        tables = _tables(b, n_bits)
        model_insert(tables, _random_sig(rs, 5, k), b, r, n_bits, n_hashes)
        batch = _copies_batch(rs, k, _random_sig(rs, 5, k), 120)
        keep, _ = model_loop(tables, batch, b, r, n_bits, n_hashes)
        pos = model_positions(batch, b, r, n_bits, n_hashes)
        assert np.array_equal(loop_on_probe_bits(pos, _preset(tables, pos), n_bits), keep)


@needs_gxx
def test_emulated_c_abi_validation(emu_lib):
    lib = emu_lib
    k, b, r, n_bits, h = 64, 8, 8, 5003, 3
    sig = np.zeros((4, k), dtype=np.uint32)
    tab = _tables(b, n_bits)
    keep = np.zeros(4, dtype=np.uint8)
    need = lib.dsk_bloom_unique_workspace_size(4, k, b, r, h)
    e = 4 * b * h
    assert need >= 32 * e + 12 * 4 and need <= 32 * e + 12 * 4 + 8 * 256
    for args in [(0, k, b, r, h), (-1, k, b, r, h), (4, k, b, 9, h), (4, k, 0, r, h), (4, k, b, r, 0), (4, k, b, r, 65),
                 (1 << 30, k, b, r, h)]:
        assert lib.dsk_bloom_unique_workspace_size(*args) == 0, args
    assert lib.dsk_bloom_unique_workspace_size((1 << 30) // (b * h), k, b, r, h) > 0
    ws = np.zeros(need // 8 + 4, dtype=np.uint64)
    p, t, wsp, kp = sig.ctypes.data, tab.ctypes.data, ws.ctypes.data, keep.ctypes.data

    def call(sig_p=p, n=4, kk=k, bb=b, rr=r, tab_p=t, words=tab.shape[1], nb=n_bits, hh=h, ws_p=wsp, wsb=need, keep_p=kp):
        return lib.dsk_bloom_unique(sig_p, n, kk, bb, rr, tab_p, words, nb, hh, ws_p, wsb, keep_p, None)

    assert call() == DSK_OK
    assert call(n=0, sig_p=None, ws_p=None, keep_p=None, wsb=0) == DSK_OK
    bad = [dict(n=-1), dict(bb=0), dict(rr=0), dict(bb=9), dict(kk=0), dict(tab_p=None), dict(hh=0), dict(hh=65),
           dict(nb=0), dict(words=1), dict(sig_p=None), dict(ws_p=None), dict(keep_p=None), dict(wsb=need - 1),
           dict(nb=(1 << 64) // b, words=((1 << 64) // b + 31) // 32), dict(tab_p=t + 2)]
    for kw in bad:
        assert call(**kw) == DSK_ERR_INVALID, kw
        assert lib.dsk_last_error()
    assert call(sig_p=p + 2) == DSK_ERR_ALIGN
    assert call(ws_p=wsp + 8, wsb=need) == DSK_ERR_ALIGN
    big = (1 << 30) // (b * h) + 1
    assert call(n=big) == DSK_ERR_INVALID


def test_thread_sanitizer_resolution():
    """The resolution under ThreadSanitizer (tests/emu/emu_tsan_bloom_unique_main.cpp, linked with the whole emulated
    library): statuses written and read by concurrent lanes through relaxed atomics, band-level drift chains resolved
    over many rounds of the single resolving CTA, checked against a serial loop."""
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = os.path.join(EMU, "_build")
    os.makedirs(out, exist_ok=True)
    exe = os.path.join(out, "emu_tsan_bloom_unique")
    build = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-ffp-contract=off", "-fsanitize=thread", "-DDSK_EMU",
                            "-I" + EMU, "-o", exe, os.path.join(EMU, "emu_capi.cpp"),
                            os.path.join(EMU, "emu_tsan_bloom_unique_main.cpp")], capture_output=True, text=True)
    if build.returncode != 0:
        pytest.skip("ThreadSanitizer build unavailable: " + build.stderr[-300:])
    env = dict(os.environ, TSAN_OPTIONS="history_size=7 halt_on_error=1 exitcode=66")
    run = subprocess.run([exe], capture_output=True, text=True, env=env, timeout=1800)
    assert "ThreadSanitizer" not in run.stderr, run.stderr[-3000:]
    assert run.returncode == 0, run.stdout + run.stderr[-2000:]
    assert run.stdout.count("identical") == 2, run.stdout


# ---- GPU: the Python API ---------------------------------------------------------------------------------------------
def _bloom(**kw):
    import datasketch_b200 as dsk
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return dsk.MinHashLSHBloom(**kw)


def _host_bits(t):
    return t.cpu().numpy().view(np.uint32)


def _gpu_bloom_for(b, r, k, n_bits, n_hashes):
    """A MinHashLSHBloom whose geometry is overridden to (b, r, n_bits, n_hashes)."""
    import torch
    bl = _bloom(threshold=0.5, num_perm=k, n=10, fp=0.5, params=(2, 1))
    bl.b, bl.r, bl.n_bits, bl.n_hashes = b, r, n_bits, n_hashes
    bl.words_per_table = _words(n_bits)
    bl._bits = torch.zeros((b, bl.words_per_table), dtype=torch.int32, device="cuda")
    return bl


def _check_gpu(bl, batch, to_host=True):
    """bl.insert_unique(batch) == the loop over the model; returns keep"""
    import torch
    before = _host_bits(bl._bits)
    want_keep, want_tables = model_loop(before, batch, bl.b, bl.r, bl.n_bits, bl.n_hashes)
    keep = bl.insert_unique(batch, to_host=to_host)
    if not to_host:
        assert keep.is_cuda and keep.dtype == torch.bool
        keep = keep.cpu().numpy()
    assert np.array_equal(keep, want_keep), np.flatnonzero(keep != want_keep)[:20]
    got = _host_bits(bl._bits)
    assert np.array_equal(got, want_tables)
    again = torch.from_numpy(before.view(np.int32).copy()).cuda()
    saved, bl._bits = bl._bits, again
    if keep.any():
        bl.insert_batch(np.asarray(batch)[keep])
    bl._bits = saved
    assert torch.equal(again, saved)
    return keep


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_device_geometries(cfg):
    k, b, r, n_bits, n_hashes = cfg
    rs = np.random.RandomState(3 * k + b)
    n = _sms() * 8 * 8 + 301 if k <= 4096 else 300       # more rows than one probe grid (SMs x 8 CTAs x 8 warps)
    bl = _gpu_bloom_for(b, r, k, n_bits, n_hashes)
    prior = _random_sig(rs, 50, k)
    bl.insert_batch(prior)
    keep = _check_gpu(bl, _copies_batch(rs, k, prior, n))
    assert not keep.all() and (keep.any() or n_bits < 1000)


@pytest.mark.gpu
def test_device_copies_chain_union_and_repeats():
    rs = np.random.RandomState(31)
    bl = _gpu_bloom_for(9, 13, 128, 1 << 20, 7)
    prior = _random_sig(rs, 100, 128)
    bl.insert_batch(prior)
    batch = _random_sig(rs, 900, 128)
    batch[100:700] = batch[50]
    batch[20:40] = prior[:20]
    keep = _check_gpu(bl, batch)
    assert keep[50] and not keep[100:700].any() and not keep[20:40].any()
    chain = _gpu_bloom_for(4, 8, 32, 1 << 22, 3)
    keep = _check_gpu(chain, _drift_chain(rs, 2100, 32, 4, 8))
    assert keep.tolist() == [j % 2 == 0 for j in range(2100)]
    for n_bits, n_hashes in TINY:   # the emulation's cases: each has all three kinds of coverage
        tiny = _gpu_bloom_for(4, 4, 16, n_bits, n_hashes)
        prior, batch = _tiny_case(n_bits, n_hashes)
        tiny.insert_batch(prior)
        t0 = _host_bits(tiny._bits)
        keep = _check_gpu(tiny, batch)
        assert all(c > 0 for c in _coverage_kinds(t0, batch, keep, 4, 4, n_bits, n_hashes))
    _check_gpu(_gpu_bloom_for(2, 15, 30, 100, 64), _random_sig(rs, 80, 30))


@pytest.mark.gpu
def test_device_batches_inputs_and_persistence(tmp_path):
    import torch
    rs = np.random.RandomState(37)
    bl = _bloom(threshold=0.8, num_perm=128, n=20000, fp=0.01, save_dir=str(tmp_path / "idx"))
    assert bl.insert_unique(np.zeros((0, 128), dtype=np.uint32)).shape == (0,)
    assert bl.insert_unique(np.zeros((0, 128), dtype=np.uint32), to_host=False).shape == (0,)
    a = _copies_batch(rs, 128, _random_sig(rs, 5, 128), 3000)
    keep_a = _check_gpu(bl, a.astype(np.uint64))                    # numpy uint64 input
    assert not _check_gpu(bl, a).any()                              # the same batch twice: nothing new
    assert not _check_gpu(bl, a[keep_a][::-1].copy()).any()         # all dropped
    bb = _copies_batch(rs, 128, a, 2000)
    d_bb = torch.from_numpy(bb.view(np.int32).copy()).cuda()         # CUDA int32 input, to_host=False
    want_keep, _ = model_loop(_host_bits(bl._bits), bb, bl.b, bl.r, bl.n_bits, bl.n_hashes)
    keep_b = bl.insert_unique(d_bb, to_host=False)
    assert keep_b.is_cuda and keep_b.dtype == torch.bool
    assert np.array_equal(keep_b.cpu().numpy(), want_keep)
    whole = _bloom(threshold=0.8, num_perm=128, n=20000, fp=0.01)
    assert np.array_equal(whole.insert_unique(np.concatenate([a, bb])), np.concatenate([keep_a, want_keep]))
    assert torch.equal(whole._bits, bl._bits)                       # A then B == A ++ B
    bl.sync()
    again = _bloom(threshold=0.8, num_perm=128, n=20000, fp=0.01, save_dir=str(tmp_path / "idx"))
    assert torch.equal(again._bits, bl._bits)
    assert not again.insert_unique(np.concatenate([a, bb])).any()


@pytest.mark.gpu
def test_device_equals_the_row_by_row_loop():
    """insert_unique == the class's own query / insert loop, row by row"""
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(41)
    kw = dict(threshold=0.8, num_perm=128, n=5000, fp=0.001)
    one, many = _bloom(**kw), _bloom(**kw)
    prior = _random_sig(rs, 1000, 128)
    one.insert_batch(prior)
    many.insert_batch(prior)
    batch = _copies_batch(rs, 128, prior, 3000)
    keep = np.zeros(len(batch), dtype=bool)
    for j, row in enumerate(batch):
        m = dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64))
        if not one.query(m):
            one.insert(m)
            keep[j] = True
    assert np.array_equal(many.insert_unique(batch), keep)
    assert torch.equal(one._bits, many._bits)


@pytest.mark.gpu
def test_device_probe_positions_above_two_to_the_32():
    import torch
    n_bits, b, r, n_hashes, n = 5 << 30, 2, 10, 4, 20_000
    if torch.cuda.mem_get_info()[0] < (4 << 30):
        pytest.skip("needs 4 GB of free device memory")
    rs = np.random.RandomState(43)
    bl = _gpu_bloom_for(b, r, b * r, n_bits, n_hashes)   # 2 x 671 MB
    try:
        prior = _random_sig(rs, 2000, b * r)
        bl.insert_batch(prior)
        batch = _copies_batch(rs, b * r, prior, n)
        pos = model_positions(batch, b, r, n_bits, n_hashes)
        assert 0.15 < (pos >= U64(1 << 32)).mean() < 0.25
        ppos = model_positions(prior, b, r, n_bits, n_hashes)
        pkeys = set((ppos + (np.arange(b, dtype=np.uint64) * U64(n_bits))[None, :, None]).ravel().tolist())
        keys = pos + (np.arange(b, dtype=np.uint64) * U64(n_bits))[None, :, None]
        preset = np.isin(keys, np.array(sorted(pkeys), dtype=np.uint64))
        want = loop_on_probe_bits(pos, preset, n_bits)
        keep = bl.insert_unique(batch)
        assert np.array_equal(keep, want)
        # the tables hold exactly the prior rows' and the kept rows' bits
        ref = torch.zeros_like(bl._bits)
        saved, bl._bits = bl._bits, ref
        bl.insert_batch(np.concatenate([prior, batch[keep]]))
        bl._bits = saved
        assert torch.equal(ref, saved)
        del ref
    finally:
        del bl
        torch.cuda.empty_cache()
