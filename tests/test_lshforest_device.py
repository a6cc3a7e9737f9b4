"""forest_query_kernel at its limits (SURVEY.md section 8 f2), against the host ``MinHashLSHForest``, which
``test_lshforest.py`` pins to the reference's own results (tests/golden/forest.npz).  Result SETS are compared, as
there.

The kernel puts one warp on a query and walks prefixes r = k..1, trees 0..l-1 in passes of 32 lanes, with a grid-stride
loop over queries.  Covered here: more queries than one grid holds, top-k lists that fill in the middle of a tree at
several r (buckets larger than top-k), top-k up to the C-ABI limit of 1024, l past one pass of 32 lanes, k = 1,
num_perm = 1, l*k < num_perm with the unused columns randomised, an empty index, re-indexing, and the input types.

CPU part: the C-ABI on the emulated library (2 SMs, 8 CTAs of 4 warps per SM: 64 queries per grid), with the tree
orders built by ``np.lexsort``.  GPU part: ``GpuLSHForest``."""
import shutil

import numpy as np
import pytest


@pytest.fixture(scope="module")
def dsk():
    import datasketch_b200
    return datasketch_b200


def _lean(dsk, row):
    return dsk.LeanMinHash(seed=1, hashvalues=row.astype(np.uint64))


def _host_forest(dsk, sig, l):
    f = dsk.MinHashLSHForest(num_perm=sig.shape[1], l=l)
    for i, row in enumerate(sig):
        f.add(i, _lean(dsk, row))
    f.index()
    return f


def _host_query(dsk, f, row, topk):
    return sorted(f.query(_lean(dsk, row), topk))


def _sets(out):
    return [sorted(int(x) for x in row if x >= 0) for row in out]


def _low_entropy(rs, n, k, dup=0):
    """values 0..2: long shared prefixes, large buckets at every r"""
    sig = rs.randint(0, 3, size=(n, k)).astype(np.uint32)
    if dup:
        sig[rs.randint(0, n, dup)] = sig[rs.randint(0, n, dup)]
    return sig


def _well_formed(out, n):
    """each row: distinct document numbers in [0, n), then -1 padding"""
    for row in out:
        got = row[row >= 0]
        assert len(set(got.tolist())) == len(got) and (got < n).all()
        assert (row[len(got):] == -1).all()


# ---- CPU: the emulated library ---------------------------------------------------------------------------------------
def _orders(sig, l, kk):
    n = len(sig)
    return np.ascontiguousarray(np.stack([np.lexsort([np.arange(n)] + [sig[:, t * kk + c] for c in range(kk - 1, -1, -1)])
                                          for t in range(l)]).astype(np.int32).reshape(l, n))


def _emu_query(lib, sig, l, q, topk):
    n, K = sig.shape
    kk = K // l
    q = np.ascontiguousarray(q)
    out = np.full((len(q), topk), -7, dtype=np.int32)
    if n:
        sig = np.ascontiguousarray(sig)
        order = _orders(sig, l, kk)
        rc = lib.dsk_forest_query(sig.ctypes.data, order.ctypes.data, n, K, l, kk, q.ctypes.data, len(q), topk,
                                  out.ctypes.data, None)
    else:
        rc = lib.dsk_forest_query(None, None, 0, K, l, kk, q.ctypes.data, len(q), topk, out.ctypes.data, None)
    assert rc == 0
    _well_formed(out, n)
    return out


needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@needs_gxx
def test_emulated_grid_stride_loop_and_topk(emu_lib, dsk):
    lib = emu_lib
    rs = np.random.RandomState(31)
    K, l, n = 32, 4, 1500
    sig = _low_entropy(rs, n, K, dup=100)
    f = _host_forest(dsk, sig, l)
    nq = 3 * (2 * 8 * 4) + 5                           # three sweeps of the emulated grid and a tail
    q = np.concatenate([sig[:nq - 40], _low_entropy(rs, 40, K)])
    for topk in (1, 31, 32, 33, 1024):
        out = _emu_query(lib, sig, l, q, topk)
        step = 1 if topk < 1024 else 9
        for j in range(0, nq, step):
            assert _sets(out[j:j + 1])[0] == _host_query(dsk, f, q[j], topk), (topk, j)
        if topk == 33:                                 # the same rows in launches of at most 4 queries
            small = np.concatenate([_emu_query(lib, sig, l, q[a:a + 4], topk) for a in range(0, nq, 4)])
            assert _sets(small) == _sets(out)
    assert ((out >= 0).sum(axis=1) == 1024).all()       # every list filled to the C-ABI limit
    bad = np.zeros((1, 1), dtype=np.int32)
    order = _orders(sig, l, K // l)
    assert lib.dsk_forest_query(sig.ctypes.data, order.ctypes.data, n, K, l, K // l, q.ctypes.data, 1, 1025,
                                bad.ctypes.data, None) != 0


@needs_gxx
@pytest.mark.parametrize("K,l", [(99, 33), (80, 40), (40, 40), (1, 1), (100, 8)])
def test_emulated_shapes(emu_lib, dsk, K, l):
    lib = emu_lib
    rs = np.random.RandomState(K + l)
    n = 400
    sig = _low_entropy(rs, n, K, dup=30)
    f = _host_forest(dsk, sig, l)
    q = np.concatenate([sig[:30], _low_entropy(rs, 20, K)])
    for topk in (1, 7, 60):
        out = _emu_query(lib, sig, l, q, topk)
        for j, row in enumerate(q):
            assert _sets(out[j:j + 1])[0] == _host_query(dsk, f, row, topk), (K, l, topk, j)
        used = l * (K // l)
        if used < K:                                   # columns past l*k are never read
            sig2, q2 = sig.copy(), q.copy()
            sig2[:, used:] = rs.randint(0, 1 << 32, size=(n, K - used), dtype=np.uint64).astype(np.uint32)
            q2[:, used:] = rs.randint(0, 1 << 32, size=(len(q), K - used), dtype=np.uint64).astype(np.uint32)
            assert _sets(_emu_query(lib, sig2, l, q2, topk)) == _sets(out)


@needs_gxx
def test_emulated_empty_index(emu_lib):
    q = np.random.RandomState(5).randint(0, 3, size=(70, 16)).astype(np.uint32)
    assert (_emu_query(emu_lib, np.zeros((0, 16), dtype=np.uint32), 4, q, 33) == -1).all()


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev_forest(dsk, sig, l):
    dev = dsk.GpuLSHForest(num_perm=sig.shape[1], l=l)
    dev.add(sig)
    dev.index()
    return dev


@pytest.mark.gpu
def test_grid_stride_loop_over_queries(dsk):
    import torch
    rs = np.random.RandomState(41)
    K, l, n = 32, 4, 3000
    sig = _low_entropy(rs, n, K, dup=200)
    dev = _dev_forest(dsk, sig, l)
    nq = 3 * (_sms() * 8 * 4) + 5                      # three grids of SMs x 8 CTAs x 4 warps and a tail
    q = np.concatenate([sig, _low_entropy(rs, nq - n, K)]) if nq > n else _low_entropy(rs, nq, K)
    d_q = torch.from_numpy(q.view(np.int32)).cuda()
    f = _host_forest(dsk, sig, l)
    for topk in (10, 33):
        out = dev.query(q, topk)
        assert out.shape == (nq, topk)
        _well_formed(out, n)
        small = torch.cat([dev.query(d_q[a:a + 4], topk, to_host=False) for a in range(0, nq, 4)]).cpu().numpy()
        assert _sets(small) == _sets(out), topk
        for j in range(0, nq, max(1, nq // 600)):      # >= 500 rows against the host class, across every grid
            assert _sets(out[j:j + 1])[0] == _host_query(dsk, f, q[j], topk), (topk, j)


@pytest.mark.gpu
def test_topk_from_1_to_the_limit(dsk):
    rs = np.random.RandomState(43)
    K, l, n = 32, 4, 3000
    sig = _low_entropy(rs, n, K, dup=200)
    dev = _dev_forest(dsk, sig, l)
    f = _host_forest(dsk, sig, l)
    q = np.concatenate([sig[:60], _low_entropy(rs, 40, K)])
    for topk in (1, 31, 32, 33, 1024):
        out = dev.query(q, topk)
        _well_formed(out, n)
        for j, row in enumerate(q):
            assert _sets(out[j:j + 1])[0] == _host_query(dsk, f, row, topk), (topk, j)
    assert ((out >= 0).sum(axis=1) == 1024).all()       # every list filled to the limit
    with pytest.raises(ValueError):
        dev.query(q, 1025)
    with pytest.raises(ValueError):
        dev.query(q, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("K,l", [(99, 33), (80, 40), (40, 40), (1, 1), (100, 8)])
def test_shapes(dsk, K, l):
    rs = np.random.RandomState(K * 7 + l)
    n = 1200
    sig = _low_entropy(rs, n, K, dup=80)
    dev = _dev_forest(dsk, sig, l)
    f = _host_forest(dsk, sig, l)
    q = np.concatenate([sig[:60], _low_entropy(rs, 40, K)])
    used = l * (K // l)
    for topk in (1, 7, 100):
        out = dev.query(q, topk)
        _well_formed(out, n)
        for j, row in enumerate(q):
            assert _sets(out[j:j + 1])[0] == _host_query(dsk, f, row, topk), (K, l, topk, j)
        if used < K:
            sig2, q2 = sig.copy(), q.copy()
            sig2[:, used:] = rs.randint(0, 1 << 32, size=(n, K - used), dtype=np.uint64).astype(np.uint32)
            q2[:, used:] = rs.randint(0, 1 << 32, size=(len(q), K - used), dtype=np.uint64).astype(np.uint32)
            assert _sets(_dev_forest(dsk, sig2, l).query(q2, topk)) == _sets(out)


@pytest.mark.gpu
def test_index_lifecycle(dsk):
    rs = np.random.RandomState(47)
    K, l = 64, 8
    q = _low_entropy(rs, 50, K)
    empty = dsk.GpuLSHForest(num_perm=K, l=l)
    with pytest.raises(ValueError):
        empty.query(q, 3)                              # index() has not been called
    empty.index()
    assert empty.is_empty() and len(empty) == 0
    assert (empty.query(q, 33) == -1).all()
    sig = _low_entropy(rs, 900, K, dup=50)
    dev = _dev_forest(dsk, sig, l)
    once = dev.query(q, 20)
    dev.index()
    assert np.array_equal(dev.query(q, 20), once)      # a second index() changes nothing
    grown = dsk.GpuLSHForest(num_perm=K, l=l)
    grown.add(sig[:300])
    grown.index()
    grown.add(sig[300:700])
    grown.add(sig[700:])
    grown.index()
    assert len(grown) == len(sig)
    f = _host_forest(dsk, sig, l)
    for topk in (1, 20, 200):
        got, fresh = grown.query(q, topk), _dev_forest(dsk, sig, l).query(q, topk)
        assert _sets(got) == _sets(fresh)
        for j, row in enumerate(q):
            assert _sets(got[j:j + 1])[0] == _host_query(dsk, f, row, topk), (topk, j)


@pytest.mark.gpu
def test_input_types(dsk):
    import torch
    rs = np.random.RandomState(53)
    K, l = 64, 8
    sig = _low_entropy(rs, 700, K, dup=50)
    sig[::5] = rs.randint(0, 1 << 32, size=(len(sig[::5]), K), dtype=np.uint64).astype(np.uint32)   # top bit set
    q = np.concatenate([sig[:40], _low_entropy(rs, 20, K)])
    want = _dev_forest(dsk, sig, l).query(q, 25)
    d_sig, d_q = torch.from_numpy(sig.view(np.int32)).cuda(), torch.from_numpy(q.view(np.int32)).cuda()
    dev = dsk.GpuLSHForest(num_perm=K, l=l)
    dev.add(d_sig[:300])
    dev.add(sig[300:].astype(np.uint64))               # numpy uint64 values that fit 32 bits are accepted
    dev.index()
    assert np.array_equal(dev.query(d_q, 25), want)
    assert np.array_equal(dev.query(q.astype(np.uint64), 25), want)
    f = _host_forest(dsk, sig, l)
    for j, row in enumerate(q):
        assert _sets(want[j:j + 1])[0] == _host_query(dsk, f, row, 25), j
    # 64-bit tensors (e.g. the int64 signatures of engine.bulk_signatures_device) are refused, not misread
    with pytest.raises(TypeError):
        dev.query(d_q.to(torch.int64) & 0xFFFFFFFF, 25)
    mixed = dsk.GpuLSHForest(num_perm=K, l=l)
    mixed.add(d_sig[:300])
    with pytest.raises(TypeError):
        mixed.add(d_sig[300:].to(torch.int64) & 0xFFFFFFFF)
    assert len(mixed) == 300
