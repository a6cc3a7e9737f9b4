"""GpuLSHForest(weighted=True): weighted MinHash signatures in the device forest (DESIGN.md section 4j).

Rows are packed as GpuLSH(weighted=True) packs them (sample j = word 2j = k as uint32, word 2j + 1 = t as int32); compared
as unsigned words they sort like the reference's big-endian (k, t) keys, so tree orders from ``np.lexsort`` over the
packed words and a walk that steps whole samples give the reference's query sets.  CPU part: the C-ABI on the emulated
library against tests/golden/forest_ranked.npz (the reference's MinHashLSHForest over WeightedMinHashGenerator
signatures, with negative t in config w2 and l * k < sample_size in w3) and against this package's host
MinHashLSHForest fed WeightedMinHash objects.  GPU part: the class, the reference's TestWeightedMinHashLSHForest
scenarios, the device signature path and the errors."""
import shutil

import numpy as np
import pytest

from test_lshforest_topk import Forest, _host, _obj, pack

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
WEIGHTED = ("w0", "w1", "w2", "w3")


@pytest.fixture(scope="module")
def dsk():
    import datasketch_b200
    return datasketch_b200


def _sets(out):
    return [sorted(int(x) for x in row if x >= 0) for row in out]


def _fixture_sets(g, key):
    return [sorted(int(x) for x in row if x >= 0) for row in g[key]]


def test_alias_and_order_argument(dsk):
    assert dsk.WeightedMinHashLSHForest is dsk.MinHashLSHForest
    assert "WeightedMinHashLSHForest" in dsk.__all__
    # unsigned word order of the packing == byte order of the reference's big-endian int64 (k, t) keys
    rs = np.random.RandomState(3)
    hv = np.stack([rs.randint(0, 5, size=(400, 3)), rs.randint(-4, 4, size=(400, 3))], axis=-1)
    hv[::7, :, 0] = (1 << 32) - 1 - rs.randint(0, 2, size=(len(hv[::7]), 3))
    keys = [bytes(h.astype(np.int64).byteswap().data) for h in hv]
    words = pack(hv)
    by_words = np.lexsort([words[:, c] for c in range(words.shape[1] - 1, -1, -1)])
    assert [keys[i] for i in by_words] == sorted(keys)


@needs_gxx
@pytest.mark.parametrize("name", WEIGHTED)
def test_emulated_query_sets(emu_lib, golden, dsk, name):
    g = golden("forest_ranked")
    ss, l, _ = (int(x) for x in g[name + "_params"])
    f = Forest(pack(g[name + "_hv"]), ss, l, True)
    q = pack(g[name + "_qhv"])
    n_self = int(g["n_self"])
    h = _host(dsk, f)
    for topk in (1, 5, 20, 200):
        got = _sets(f.query(emu_lib, q, topk))
        assert got == _fixture_sets(g, "%s_qset%d" % (name, topk)), topk
        assert _sets(f.query(emu_lib, f.words[:n_self], topk)) == _fixture_sets(g, "%s_sset%d" % (name, topk)), topk
        assert got == [sorted(h.query(_obj(dsk, f, row), topk)) for row in q], topk   # the host class on WeightedMinHash
    if name == "w2":                                   # weights of about 1e-6: every t is negative
        assert (g[name + "_hv"][..., 1] < 0).all() and (g[name + "_qhv"][..., 1] < 0).all()


@needs_gxx
def test_emulated_walk_steps_samples(emu_lib, dsk):
    """Rows that agree on a sample's k but not its t: a word-by-word walk would see a longer prefix than the
    reference does and fill the list differently."""
    rs = np.random.RandomState(5)
    n, ss, l = 300, 12, 3
    hv = np.stack([np.zeros((n, ss), np.int64) + rs.randint(0, 2, size=(n, ss)), rs.randint(-2, 2, size=(n, ss))], -1)
    f = Forest(pack(hv), ss, l, True)
    h = _host(dsk, f)
    q = f.words[:80]
    for topk in (1, 3, 10, 40):
        assert _sets(f.query(emu_lib, q, topk)) == [sorted(h.query(_obj(dsk, f, row), topk)) for row in q], topk


# ---- GPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", WEIGHTED)
def test_fixture_query_sets_through_the_class(golden, dsk, name):
    import torch
    g = golden("forest_ranked")
    ss, l, _ = (int(x) for x in g[name + "_params"])
    hv, qhv = g[name + "_hv"], g[name + "_qhv"]
    dev = dsk.GpuLSHForest(num_perm=ss, l=l, weighted=True)
    dev.add(hv[:100])
    dev.add(torch.from_numpy(hv[100:]).cuda())
    dev.index()
    assert len(dev) == len(hv)
    n_self = int(g["n_self"])
    for topk in (1, 5, 20, 200):
        assert _sets(dev.query(qhv, topk)) == _fixture_sets(g, "%s_qset%d" % (name, topk))
        assert _sets(dev.query(hv[:n_self], topk)) == _fixture_sets(g, "%s_sset%d" % (name, topk))
    wm = [dsk.WeightedMinHash(1, h) for h in qhv]
    assert _sets(dev.query(wm, 20)) == _fixture_sets(g, "%s_qset20" % name)
    assert [sorted(x) for x in dev.query_keys(qhv[:3], 5)] == _fixture_sets(g, "%s_qset5" % name)[:3]


@pytest.mark.gpu
def test_reference_scenarios(dsk):
    """TestWeightedMinHashLSHForest (the reference's test/test_lshforest.py): every indexed key is in its own top-10
    set, and a repeated add / index behaves as on an unweighted forest."""
    mg = dsk.WeightedMinHashGenerator(10, 128, seed=1)
    rs = np.random.RandomState(7)
    data = rs.randint(0, 10, size=(40, 10)).astype(np.float64) + 1
    hv = np.stack([mg.minhash(v).hashvalues for v in data])
    keys = ["k%d" % i for i in range(len(hv))]
    dev = dsk.GpuLSHForest(num_perm=128, l=8, weighted=True)
    dev.add(hv[:20], keys[:20])
    dev.index()
    dev.add(hv[20:], keys[20:])
    dev.index()
    assert not dev.is_empty()
    for i, row in enumerate(dev.query_keys(hv, 10)):
        assert keys[i] in row and len(row) <= 10
    again = dev.query(hv, 10)
    dev.index()
    assert np.array_equal(dev.query(hv, 10), again)


@pytest.mark.gpu
def test_device_signatures(dsk):
    mg = dsk.WeightedMinHashGenerator(64, 64, seed=3)
    rs = np.random.RandomState(9)
    X = (rs.randint(1, 20, size=(500, 64)) * (rs.rand(500, 64) >= 0.6)).astype(np.float32)
    X[:, 0] += 1
    X[250:] = X[:250] * (1 + (rs.rand(250, 64) < 0.1))
    host = mg.minhash_batch(X)
    d_hv = mg.minhash_batch(X, to_host=False)
    a = dsk.GpuLSHForest(num_perm=64, l=8, weighted=True)
    a.add(host)
    a.index()
    b = dsk.GpuLSHForest(num_perm=64, l=8, weighted=True)
    b.add(d_hv)
    b.index()
    for topk in (1, 10, 100):
        assert np.array_equal(a.query(host, topk), b.query(d_hv, topk))
    assert all(np.array_equal(x, y) for x, y in zip(a.query_topk(host, 7, 30), b.query_topk(d_hv, 7, 30)))
    assert all(np.array_equal(x, y) for x, y in zip(a.neighbors(7, 30), b.neighbors(7, 30)))


@pytest.mark.gpu
def test_errors_leave_the_forest_unchanged(dsk):
    rs = np.random.RandomState(11)
    hv = np.stack([rs.randint(0, 9, size=(30, 16)), rs.randint(-3, 3, size=(30, 16))], -1)
    dev = dsk.GpuLSHForest(num_perm=16, l=4, weighted=True)
    dev.add(hv)
    for bad in (hv[:, :, 0], hv[:, :8], hv.astype(np.float64), np.concatenate([hv[:1], hv[:1] * 0 - 1]),
                np.stack([hv[..., 0], hv[..., 1] + (1 << 31)], -1)):
        with pytest.raises((ValueError, TypeError)):
            dev.add(bad)
    assert len(dev) == 30
    with pytest.raises(ValueError):
        dev.query(hv, 3)                                # index() has not been called
    dev.index()
    with pytest.raises(ValueError):
        dev.query(hv[:, :, 0], 3)
    plain = dsk.GpuLSHForest(num_perm=16, l=4)
    with pytest.raises(ValueError):
        plain.add(hv)                                   # a 3-D array on an unweighted forest
    assert len(plain) == 0
