"""Weighted MinHash on sparse rows: ``dsk_wmh_minhash_csr`` (wmh_csr_kernel) and the scipy.sparse / torch.sparse_csr
inputs of ``WeightedMinHashGenerator.minhash_batch`` and ``minhash_many``.

Every case runs twice: on the emulated library through the C-ABI (CPU suite; the host side is the module's own
``_csr_arrays`` and numpy's float32 log, as ``minhash_batch`` prepares a scipy matrix) and on the H100 through the Python
API (``-m gpu``).  The expectation is always the densified rows: ``oracle_np.wmh_from_log`` of numpy's float32 log of
``X.tocsr().toarray()`` cast to float32, with no tolerance, or the reference's own results in tests/golden/wmh_sparse.npz
(oracle/gen_golden_wmh_sparse.py) and tests/golden/wmh_special.npz.
"""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle_np as o

WMH_MANY, WMH_INPUT_LOG = 1, 2
INT64_MIN = np.iinfo(np.int64).min
TILE = 512                    # entries wmh_csr_kernel stages per tile


def _log32(V):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(np.asarray(V, dtype=np.float32))


def _log64to32(V):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(np.asarray(V, dtype=np.float32).astype(np.float64)).astype(np.float32)


def _dense32(X):
    return np.asarray(X.tocsr().toarray(), dtype=np.float32)


def _want(X, par, many):
    """(out, status) of the densified rows with numpy's float32 log."""
    return o.wmh_from_log(_log32(_dense32(X)), *par, many=many)


class _Emu:
    """The emulated library through the C-ABI; host preparation as minhash_batch does it."""
    name = "emu"

    def __init__(self, lib):
        self.lib = lib
        self.sm_count = 2
        self._gens = []

    def handle(self, par):
        for p, h in self._gens:
            if p is par:
                return h
        rs, lc, be = (np.ascontiguousarray(x, dtype=np.float32) for x in par)
        h = ctypes.c_void_p()
        assert self.lib.dsk_wmh_create(rs.ctypes.data, lc.ctypes.data, be.ctypes.data, rs.shape[0], rs.shape[1], 0,
                                       ctypes.byref(h)) == 0
        self._gens.append((par, h))
        return h

    def raw(self, par, indptr, cols, vals, flags):
        ss = par[0].shape[0]
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        n = len(indptr) - 1
        cols = np.ascontiguousarray(cols, dtype=np.int32) if len(cols) else np.zeros(1, np.int32)
        vals = np.ascontiguousarray(vals, dtype=np.float32) if len(vals) else np.zeros(1, np.float32)
        out = np.full((n, ss, 2), -7, dtype=np.int64)
        st = np.full(n, -7, dtype=np.int32)
        rc = self.lib.dsk_wmh_minhash_csr(self.handle(par), indptr.ctypes.data, cols.ctypes.data, vals.ctypes.data,
                                          ctypes.c_int64(n), out.ctypes.data, st.ctypes.data, flags, None)
        assert rc == 0, self.lib.dsk_last_error()
        return out, st

    def sample(self, par, X, many):
        from datasketch_b200.weighted_minhash import _csr_arrays
        indptr, cols, w = _csr_arrays(X, par[0].shape[1])
        return self.raw(par, indptr, cols, _log32(w), WMH_INPUT_LOG | int(many))

    def close(self):
        for _, h in self._gens:
            self.lib.dsk_wmh_destroy(h)


class _Gpu:
    """The Python API on the device."""
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        from datasketch_b200 import _native as nv
        self.dsk = dsk
        self.sm_count = nv.device_info(0)["sm_count"]
        self._gens = []

    def gen(self, par):
        for p, g in self._gens:
            if p is par:
                return g
        g = self.dsk.WeightedMinHashGenerator(par[0].shape[1], par[0].shape[0], 1)
        g.rs, g.ln_cs, g.betas = par                     # before the device handle is built
        self._gens.append((par, g))
        return g

    def sample(self, par, X, many):
        return self.gen(par)._sample_csr(X, 0, many=many)

    def close(self):
        self._gens = []


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def run(request):
    if request.param == "emu":
        r = _Emu(request.getfixturevalue("emu_lib"))
    else:
        r = _Gpu()
    yield r
    r.close()


def _assert_api(run, par, X):
    """On the device, the public methods: minhash_batch's rows and errors, minhash_many's values and None rows."""
    if run.name != "gpu":
        return
    gen = run.gen(par)
    want, st = _want(X, par, many=False)
    if (st == 0).all():
        assert np.array_equal(gen.minhash_batch(X), want)
    else:
        with pytest.raises(ValueError if (st == 1).any() else OverflowError):
            gen.minhash_batch(X)
    want, st = _want(X, par, many=True)
    ms = gen.minhash_many(X)
    assert [m is None for m in ms] == (st == 1).tolist()
    assert all(np.array_equal(m.hashvalues, want[i]) for i, m in enumerate(ms) if m is not None)


def _random_csr(rng, lens, dim, zipf=None):
    """Rows of the given lengths, sorted distinct columns (uniform, or Zipf-distributed), lognormal weights."""
    indptr = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    cols = []
    for ln in lens:
        if zipf:
            c = np.unique((rng.zipf(zipf, 4 * ln + 8) - 1) % dim)[:ln]
            c = np.sort(np.concatenate([c, np.setdiff1d(rng.choice(dim, min(dim, 2 * ln), replace=False), c)[:ln - len(c)]]))
        else:
            c = np.sort(rng.choice(dim, ln, replace=False))
        cols.append(c)
    cols = np.concatenate(cols).astype(np.int32) if cols else np.zeros(0, np.int32)
    vals = rng.lognormal(0, 2, int(indptr[-1])).astype(np.float32)
    return sp.csr_matrix((vals, cols, indptr), shape=(len(lens), dim))


# ---- the reference's results -----------------------------------------------------------------------------------------
def test_reference_fixture(run, golden):
    """The reference's minhash_many on a dim-200,003 scipy CSR matrix, and its minhash on 24 of those rows densified."""
    g = golden("wmh_sparse")
    dim, ss, seed = (int(x) for x in g["cfg"])
    par = o.wmh_params(dim, ss, seed)
    assert np.array_equal([x.astype(np.float64).sum() for x in par], g["param_sums"])
    X = sp.csr_matrix((g["data"], g["indices"], g["indptr"]), shape=(len(g["indptr"]) - 1, dim))
    out, st = run.sample(par, X, many=True)
    null = g["many_null"]
    assert np.array_equal(st == 1, null) and not (st[~null]).any()
    assert np.array_equal(out[~null], g["many_out"][~null])
    out, st = run.sample(par, X, many=False)
    rows = g["dense_rows"]
    assert not st[rows].any() and np.array_equal(out[rows], g["dense_out"])
    assert np.array_equal(st == 1, null)
    if run.name == "gpu":
        gen = run.gen(par)
        ms = gen.minhash_many(X)
        assert [m is None for m in ms] == null.tolist()
        assert all(np.array_equal(m.hashvalues, g["many_out"][i]) for i, m in enumerate(ms) if m is not None)
        assert np.array_equal(gen.minhash_batch(X[rows]), g["dense_out"])


# ---- shapes and row lengths, host logarithm: exact ------------------------------------------------------------------
@pytest.mark.parametrize("ss", [1, 31, 32, 33, 127, 128, 129, 300])
def test_shapes_exact(run, ss):
    """Rows of 0, 1, 2, 7, 8, 9 and many entries, one longer than three tiles, explicit zeros and -0.0 stored."""
    dim = 3001
    rng = np.random.RandomState(ss)
    lens = [0, 1, 2, 7, 8, 9, TILE - 1, TILE, TILE + 1, 3 * TILE + 5, 40, 0, 1]
    X = _random_csr(rng, lens, dim)
    X.data[rng.rand(X.nnz) < 0.1] = 0.0
    X.data[5] = -0.0
    X.data[X.indptr[9]:X.indptr[9] + 3] = [0.0, -0.0, 0.0]
    par = o.wmh_params(dim, ss, 5 + ss)
    for many in (False, True):
        want, wst = _want(X, par, many)
        out, st = run.sample(par, X, many)
        assert np.array_equal(st, wst) and np.array_equal(out, want), many
    assert (wst == 1).sum() == 2
    _assert_api(run, par, X[np.diff(X.indptr) > 0])


def test_long_row_ties_far_apart(run):
    """Columns far apart (and either side of a tile boundary inside one row) with equal parameters and weights tie in
    every sample: the first column wins in both modes.  The long row holds them among thousands of other entries."""
    dim, ss = 70_001, 130
    rs, lc, be = (x.copy() for x in o.wmh_params(dim, ss, 23))
    pairs = [(5, 60_000), (100, 40_000), (2, 69_999)]
    for i, j in pairs:
        rs[:, j], lc[:, j], be[:, j] = rs[:, i], lc[:, i], be[:, i]
    par = (rs, lc, be)
    rng = np.random.RandomState(3)
    rows = []
    for i, j in pairs:
        v = np.zeros(dim, np.float32)
        v[i] = v[j] = rng.uniform(0.5, 5)
        rows.append(v)
    v = np.zeros(dim, np.float32)
    v[rng.choice(dim, 5000, replace=False)] = rng.uniform(0.1, 2, 5000)
    for i, j in pairs:
        v[i] = v[j] = 1e4
    rows.append(v)
    # a tie split by a tile boundary: the row's TILE-th and (TILE + 1)-th entries
    v = np.zeros(dim, np.float32)
    cols = np.sort(rng.choice(np.arange(1000, 60_000), 2 * TILE, replace=False))
    v[cols] = rng.uniform(0.1, 2, len(cols))
    a, b = cols[TILE - 1], cols[TILE]
    rows.append(v)
    V = np.stack(rows)
    rs2, lc2, be2 = rs.copy(), lc.copy(), be.copy()
    rs2[:, b], lc2[:, b], be2[:, b] = rs2[:, a], lc2[:, a], be2[:, a]
    V[-1, b] = V[-1, a] = 1e4
    par = (rs2, lc2, be2)
    X = sp.csr_matrix(V)
    for many in (False, True):
        want, wst = _want(X, par, many)
        out, st = run.sample(par, X, many)
        assert not st.any() and np.array_equal(out, want)
        for r, (i, j) in enumerate(pairs):
            assert (out[r, :, 0] == i).all()
        assert not np.isin(out[3, :, 0], [j for _, j in pairs]).any()
        assert (out[4, :, 0] != b).all() and (out[4, :, 0] == a).mean() > 0.5
    _assert_api(run, par, X)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_special_weights(run, golden, tag):
    """NaN, +-inf, negative, subnormal and FLT_MAX weights against the reference's results, both as scipy stores them
    (no zeros) and with every zero and -0.0 stored explicitly."""
    g = golden("wmh_special")
    X = g["X"]
    dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
    par = o.wmh_params(dim, ss, seed)
    err = g[f"{tag}_err"]
    n = len(X)
    full = sp.csr_matrix((X.ravel(), np.tile(np.arange(dim), n), np.arange(0, n * dim + 1, dim)), shape=X.shape)
    assert full.nnz == X.size
    for S in (sp.csr_matrix(X), full):
        out, st = run.sample(par, S, many=True)
        null = g[f"{tag}_many_null"]
        assert np.array_equal(st == 1, null)
        assert np.array_equal(out[~null], g[f"{tag}_many_out"][~null])
        assert (out[st == 2][:, :, 1] == INT64_MIN).all()
        out, st = run.sample(par, S, many=False)
        ok = err == ""
        assert np.array_equal(out[ok], g[f"{tag}_out"][ok]) and not st[ok].any()
        assert np.array_equal(st == 1, err == "ValueError") and np.array_equal(st == 2, err == "OverflowError")
        for many in (False, True):
            want, wst = _want(S, par, many)
            o_, s_ = run.sample(par, S, many)
            assert np.array_equal(s_, wst) and np.array_equal(o_, want)
    if run.name == "gpu":
        gen = run.gen(par)
        for bad, exc in (("ValueError", ValueError), ("OverflowError", OverflowError)):
            with pytest.raises(exc):
                gen.minhash_batch(full[np.where((err == "") | (err == bad))[0]])
        assert np.array_equal(gen.minhash_batch(full[np.where(err == "")[0]]), g[f"{tag}_out"][err == ""])


def test_more_rows_than_ctas(run):
    """3 * 16 * sm_count + 5 rows: every CTA of the capped grid takes three or four rows."""
    n = 3 * 16 * run.sm_count + 5
    dim, ss = 997, 129
    rng = np.random.RandomState(9)
    lens = rng.randint(0, 60, n)
    lens[rng.choice(n, 4, replace=False)] = [0, 1, TILE + 3, 700]
    X = _random_csr(rng, lens, dim, zipf=1.1)
    par = o.wmh_params(dim, ss, 31)
    for many in (False, True):
        want, wst = _want(X, par, many)
        out, st = run.sample(par, X, many)
        assert np.array_equal(st, wst) and np.array_equal(out, want)


# ---- non-canonical scipy input: equal to the densified matrix -------------------------------------------------------
def _noncanonical_cases():
    rng = np.random.RandomState(11)
    dim = 40
    # unsorted columns
    unsorted = sp.csr_matrix((np.array([3, 1, 2, 5, 0.5, 4], np.float32), np.array([7, 2, 30, 1, 39, 0]),
                              np.array([0, 3, 3, 6])), shape=(3, dim))
    # duplicates whose float32 sum depends on the order: [1e8, -1e8, 1] sums to 1, [1, 1e8, -1e8] to 0
    dup = sp.csr_matrix((np.array([1e8, -1e8, 1, 2, 1, 1e8, -1e8, 2], np.float32),
                         np.array([4, 4, 4, 9, 4, 4, 4, 9]), np.array([0, 4, 8])), shape=(2, dim))
    # int64 data, with duplicates
    ints = sp.csr_matrix((np.array([2, 3, 1, 7, 9, 1], np.int64), np.array([5, 1, 5, 0, 3, 3]),
                          np.array([0, 3, 6])), shape=(2, dim))
    D = (rng.randint(0, 5, (6, dim)) * (rng.rand(6, dim) < 0.3)).astype(np.float32)
    D[2] = 0
    D[3, 1] = 1e-30
    coo = sp.coo_matrix(D)
    coo_dup = sp.coo_matrix((np.array([1, 1e8, -1e8, 1e8, -1e8, 1], np.float32),
                             (np.array([0, 0, 0, 1, 1, 1]), np.array([3, 3, 3, 3, 3, 3]))), shape=(2, dim))
    return [("unsorted", unsorted), ("dup", dup), ("int64", ints), ("coo", coo), ("coo_dup", coo_dup),
            ("csc", sp.csc_matrix(D)), ("csr_array", sp.csr_array(D))]


def test_csr_arrays_noncanonical():
    """_csr_arrays gives the canonical rows of exactly the densified matrix (no device needed)."""
    from datasketch_b200.weighted_minhash import _csr_arrays
    for name, X in _noncanonical_cases():
        indptr, cols, w = _csr_arrays(X, X.shape[1])
        assert indptr.dtype == np.int64 and cols.dtype == np.int32 and w.dtype == np.float32
        for i in range(X.shape[0]):
            c = cols[indptr[i]:indptr[i + 1]]
            assert (np.diff(c) > 0).all(), name
        got = np.zeros(X.shape, np.float32)
        got[np.repeat(np.arange(X.shape[0]), np.diff(indptr)), cols] = w
        assert np.array_equal(got.view(np.uint32), _dense32(X).view(np.uint32)), name
    dup = dict(_noncanonical_cases())["dup"]
    assert _dense32(dup)[0, 4] == 1 and _dense32(dup)[1, 4] == 0      # the order matters, and is kept


def test_noncanonical_input(run):
    for name, X in _noncanonical_cases():
        par = o.wmh_params(X.shape[1], 33, 2)
        for many in (False, True):
            want, wst = _want(X, par, many)
            out, st = run.sample(par, X, many)
            assert np.array_equal(st, wst) and np.array_equal(out, want), (name, many)


# ---- malformed input ------------------------------------------------------------------------------------------------
def test_malformed_scipy_refused(run):
    """Out-of-range columns and a bad indptr: ValueError before the kernel."""
    par = o.wmh_params(10, 4, 1)
    bad_cols = sp.csr_matrix((np.ones(3, np.float32), np.array([1, 2, 3]), np.array([0, 1, 3])), shape=(2, 10))
    bad_cols.indices[2] = 10
    with pytest.raises(ValueError, match="row 1"):
        run.sample(par, bad_cols, False)
    bad_cols.indices[2] = -1
    with pytest.raises(ValueError, match="row 1"):
        run.sample(par, bad_cols, True)
    bad_ptr = sp.csr_matrix((np.ones(3, np.float32), np.array([1, 2, 3]), np.array([0, 1, 3])), shape=(2, 10))
    bad_ptr.indptr[1] = 3
    bad_ptr.indptr[2] = 2
    with pytest.raises(ValueError, match="indptr"):
        run.sample(par, bad_ptr, False)
    with pytest.raises(ValueError, match="dimension"):
        run.sample(par, sp.csr_matrix((2, 11), dtype=np.float32), False)


def test_capi_status_3_and_arguments(emu_lib):
    """The kernel's own check: a row with repeated, descending or out-of-range columns gets status 3 and (0, 0); the
    other rows are unaffected.  n = 0 is a no-op; bad arguments are DSK_ERR_INVALID with a message."""
    run = _Emu(emu_lib)
    dim, ss = 4000, 40
    par = o.wmh_params(dim, ss, 3)
    rng = np.random.RandomState(1)
    X = _random_csr(rng, [5, 5, 5, 5, 5, 3 * TILE, 3 * TILE, 5], dim)
    cols = X.indices.copy()
    ip = X.indptr
    cols[ip[1] + 2] = cols[ip[1] + 1]                     # repeated
    cols[ip[2] + 3], cols[ip[2] + 4] = cols[ip[2] + 4], cols[ip[2] + 3]   # descending
    cols[ip[3]] = dim                                     # out of range
    cols[ip[5] + TILE] = cols[ip[5] + TILE - 1]           # repeated across a tile boundary
    cols[ip[6] + 2 * TILE + 7] = -5
    vlog = _log32(X.data)
    for flags in (WMH_INPUT_LOG, WMH_INPUT_LOG | WMH_MANY):
        out, st = run.raw(par, ip, cols, vlog, flags)
        assert st.tolist() == [0, 3, 3, 3, 0, 3, 3, 0]
        assert not out[st == 3].any()
        want, _ = _want(X, par, bool(flags & WMH_MANY))
        assert np.array_equal(out[st == 0], want[st == 0])
    lib = emu_lib
    h = run.handle(par)
    z = np.zeros(4, np.int64)
    assert lib.dsk_wmh_minhash_csr(h, None, None, None, ctypes.c_int64(0), None, None, 0, None) == 0
    assert lib.dsk_wmh_minhash_csr(h, z.ctypes.data, None, z.ctypes.data, ctypes.c_int64(1), z.ctypes.data,
                                   z.ctypes.data, 0, None) != 0
    assert b"dsk_wmh_minhash_csr" in lib.dsk_last_error()
    assert lib.dsk_wmh_minhash_csr(h, z.ctypes.data, z.ctypes.data, z.ctypes.data, ctypes.c_int64(-1), z.ctypes.data,
                                   z.ctypes.data, 0, None) != 0
    assert lib.dsk_wmh_minhash_csr(h, z.ctypes.data, z.ctypes.data, z.ctypes.data, ctypes.c_int64(1), z.ctypes.data,
                                   z.ctypes.data, 4, None) != 0        # unknown flags
    assert lib.dsk_wmh_minhash_csr(None, z.ctypes.data, z.ctypes.data, z.ctypes.data, ctypes.c_int64(1),
                                   z.ctypes.data, z.ctypes.data, 0, None) != 0
    run.close()


# ---- torch.sparse_csr on the device ---------------------------------------------------------------------------------
def _torch_csr(X, dtype=None, index_dtype=None):
    import torch
    X = X.tocsr()
    crow = torch.from_numpy(X.indptr.astype(index_dtype or np.int64))
    col = torch.from_numpy(X.indices.astype(index_dtype or np.int64))
    val = torch.from_numpy(np.asarray(X.data, dtype=dtype or X.data.dtype))
    return torch.sparse_csr_tensor(crow, col, val, X.shape).cuda()


@pytest.mark.gpu
def test_torch_csr_device_log():
    """A CUDA torch.sparse_csr tensor takes the device logarithm: equal to the oracle fed the float64 log rounded to
    float32 (rows near a float32 rounding midpoint exempt), and to minhash_batch of the same tensor densified."""
    import torch
    import datasketch_b200 as dsk
    dim, ss = 5003, 129
    rng = np.random.RandomState(4)
    lens = rng.randint(1, 300, 200)
    lens[:3] = [1, 2, 3 * TILE]
    X = _random_csr(rng, lens, dim, zipf=1.1)
    gen = dsk.WeightedMinHashGenerator(dim, ss, 8)
    par = (gen.rs, gen.ln_cs, gen.betas)
    D = _dense32(X)
    with np.errstate(divide="ignore", invalid="ignore"):
        l64 = np.log(X.data.astype(np.float64))
    f = l64.astype(np.float32)
    other = np.nextafter(f, np.where(l64 > f.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)))
    mid = (f.astype(np.float64) + other.astype(np.float64)) / 2
    near_e = np.abs(l64 - mid) <= 2 * np.spacing(np.abs(l64))
    near = np.zeros(len(lens), bool)
    near[np.repeat(np.arange(len(lens)), lens)[near_e]] = True
    assert near.sum() <= 2
    for T in (_torch_csr(X), _torch_csr(X, np.float64, np.int32)):
        for many in (False, True):
            want, _ = o.wmh_from_log(_log64to32(D), *par, many=many)
            got, st = gen._sample_csr(T, 0, many=many)
            assert not st.any() and np.array_equal(got[~near], want[~near]), many
        dev = gen.minhash_batch(T, to_host=False)
        assert dev.is_cuda and dev.dtype == torch.int64
        assert np.array_equal(dev.cpu().numpy(), gen.minhash_batch(T.to_dense()))
    # the host logarithm on the same rows (scipy), for comparison: the reference's exact values
    assert np.array_equal(gen.minhash_batch(X), o.wmh_from_log(_log32(D), *par)[0])
    # explicit zeros stored in a torch CSR are skipped like left-out columns
    X0 = X.copy()
    X0.data[::3] = 0
    keep = np.diff(sp.csr_matrix(_dense32(X0)).indptr) > 0
    T0 = _torch_csr(X0[np.where(keep)[0]])
    assert np.array_equal(gen.minhash_batch(T0), gen.minhash_batch(T0.to_dense()))


@pytest.mark.gpu
def test_torch_csr_malformed_refused():
    """Repeated, descending or out-of-range columns in a torch CSR row raise ValueError naming the first bad row (the
    kernel's status 3); a bad crow_indices is refused before the kernel.  n = 0 returns an empty result."""
    import torch
    import datasketch_b200 as dsk
    gen = dsk.WeightedMinHashGenerator(50, 8, 1)

    def T(crow, col, n=None):
        crow, col = torch.tensor(crow, dtype=torch.int64), torch.tensor(col, dtype=torch.int64)
        return torch.sparse_csr_tensor(crow, col, torch.ones(len(col)), (n or len(crow) - 1, 50)).cuda()

    ok = T([0, 2, 4, 5], [1, 2, 3, 40, 7])
    assert gen.minhash_batch(ok).shape == (3, 8, 2)
    for col, row in (([1, 2, 3, 3, 7], 1), ([1, 2, 40, 3, 7], 1), ([1, 2, 3, 40, 50], 2), ([2, 1, 3, 40, 7], 0),
                     ([1, 2, 3, 40, -1], 2), ([1, 2, 3, 40, 1 << 33], 2)):
        with pytest.raises(ValueError, match="row %d" % row):
            gen.minhash_batch(T([0, 2, 4, 5], col))
        with pytest.raises(ValueError, match="row %d" % row):
            gen._sample_csr(T([0, 2, 4, 5], col), 0, many=True)
    for crow in ([1, 2, 4, 5], [0, 3, 2, 5], [0, 2, 4, 6]):
        with pytest.raises(ValueError, match="crow_indices"):
            gen.minhash_batch(T(crow, [1, 2, 3, 40, 7]))
    empty = torch.sparse_csr_tensor(torch.zeros(1, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                                    torch.zeros(0), (0, 50)).cuda()
    assert gen.minhash_batch(empty).shape == (0, 8, 2)
    assert gen.minhash_many(sp.csr_matrix((0, 50), dtype=np.float32)) == []
    with pytest.raises(ValueError, match="all zeros"):
        gen.minhash_batch(T([0, 2, 2, 3], [1, 2, 7]))


# ---- at scale on the device -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scale_zipf_rows():
    """dim 2^20, ss 128, 200k Zipf rows: minhash_batch equals the dense kernel on a densified sample of rows,
    minhash_many equals the densify path on them, and a GpuLSH(weighted=True) filled from the device result of a torch
    CSR tensor answers query_jaccard as one filled from the host copy."""
    import torch
    import datasketch_b200 as dsk
    dim, ss, n = 1 << 20, 128, 200_000
    rng = np.random.RandomState(12)
    lens = np.minimum(rng.zipf(1.5, n) * 40, 5000)
    lens[rng.choice(n, 500, replace=False)] = 0
    nnz = int(lens.sum())
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=indptr[1:])
    cols = ((rng.zipf(1.1, nnz) - 1) % dim).astype(np.int64)
    rows = np.repeat(np.arange(n), lens)
    order = np.lexsort((cols, rows))
    key = rows[order] * dim + cols[order]
    first = np.ones(nnz, bool)
    first[1:] = key[1:] != key[:-1]                        # Zipf repeats: keep each (row, column) once
    key = key[first]
    vals = rng.randint(1, 50, len(key)).astype(np.float32)
    vals[::7] = rng.uniform(1e-5, 1e-2, len(vals[::7]))
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(key // dim, minlength=n), out=indptr[1:])
    X = sp.csr_matrix((vals, (key % dim).astype(np.int32), indptr), shape=(n, dim))
    empty = np.diff(indptr) == 0
    gen = dsk.WeightedMinHashGenerator(dim, ss, 1)
    sample = np.unique(np.concatenate([rng.choice(np.where(~empty)[0], 200, replace=False),
                                       np.where(~empty)[0][-5:], [int(np.argmax(np.diff(indptr)))]]))
    D = X[sample].toarray().astype(np.float32)
    ne = np.where(~empty)[0]
    got = gen.minhash_batch(X[ne])
    assert np.array_equal(got[np.searchsorted(ne, sample)], gen.minhash_batch(D))
    ms = gen.minhash_many(X)
    assert [i for i, m in enumerate(ms) if m is None] == np.where(empty)[0].tolist()
    dense_many, st = gen._sample(D, 0, many=True)
    assert not st.any()
    assert all(np.array_equal(ms[i].hashvalues, dense_many[j]) for j, i in enumerate(sample))
    T = _torch_csr(X[ne])
    dev = gen.minhash_batch(T, to_host=False)
    host = dev.cpu().numpy()
    qs = host[rng.choice(len(ne), 2000, replace=False)]
    results = []
    for sig in (dev, host):
        lsh = dsk.GpuLSH(threshold=0.5, num_perm=ss, capacity=len(ne), weighted=True)
        lsh.insert(sig)
        ptr, idx, eq = (np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x) for x in lsh.query_jaccard(qs))
        q = np.repeat(np.arange(len(qs)), np.diff(ptr))
        order = np.lexsort((idx, q))                       # candidates come in no particular order within a query
        results.append((ptr, idx[order], eq[order]))
    for a, b in zip(*results):
        assert np.array_equal(a, b)
    ptr, idx, eq = results[0]
    assert ptr[-1] >= len(qs) and (eq == ss).sum() >= len(qs)
