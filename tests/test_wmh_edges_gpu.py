"""GPU: wmh_kernel at the shapes and values where it can go wrong, compared exactly with the float32 oracle.

- shapes: sample counts around the 128-thread slice (blockIdx.y > 0, ss_pad columns), dims around the 4-dim unroll and
  the 256-dim tile (the remainder loop), 1 / 7 / 8 / 9 vectors and more vector groups than the grid has CTAs;
- host logarithm (numpy's, passed with DSK_WMH_INPUT_LOG): equal to the oracle with no tolerance;
- device logarithm (CUDA tensors, ``device_log=True``): equal to the oracle fed the float64 log rounded to float32,
  and to the numpy-log oracle up to float64-confirmed near-ties;
- constructed ties (first index wins), floor arguments at and one ulp around an integer, and special weights (zeros,
  -0.0, negative, NaN, +-inf, subnormals, FLT_MAX) against the reference's results in tests/golden/wmh_special.npz.
"""
import numpy as np
import pytest

from oracle import oracle_np as o

pytestmark = pytest.mark.gpu

WMH_MANY, WMH_INPUT_LOG = 1, 2
INT64_MIN = np.iinfo(np.int64).min


@pytest.fixture(scope="module")
def dsk():
    import datasketch_b200
    return datasketch_b200


def _log32(V):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(np.asarray(V, dtype=np.float32))


def _log64to32(V):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log(np.asarray(V, dtype=np.float32).astype(np.float64)).astype(np.float32)


def _weights(rng, n, dim, zeros=0.3):
    V = (rng.lognormal(0, 2, (n, dim)) * (rng.rand(n, dim) >= zeros)).astype(np.float32)
    V[:, rng.randint(dim)] += 0.25          # no empty row
    return V


def _raw(gen, X, flags):
    """dsk_wmh_minhash on a CUDA float32 tensor as it is: (out, status) on the host."""
    import torch
    from datasketch_b200 import _native as nv
    X = X.contiguous()
    assert X.dtype == torch.float32 and X.is_cuda
    h = gen._handle(X.device.index)
    out = torch.full((X.shape[0], gen.sample_size, 2), -7, dtype=torch.int64, device=X.device)
    st = torch.full((X.shape[0],), -7, dtype=torch.int32, device=X.device)
    nv.check(nv.load().dsk_wmh_minhash(h, X.data_ptr(), X.shape[0], out.data_ptr(), st.data_ptr(), flags,
                                       torch.cuda.current_stream(X.device).cuda_stream))
    return out.cpu().numpy(), st.cpu().numpy()


def _many_array(ms, ss):
    return np.stack([np.full((ss, 2), -1) if m is None else m.hashvalues for m in ms]).astype(np.int64)


# ---- shapes, host logarithm: exact ----------------------------------------------------------------------------------
SHAPES = [  # (ss, dim, n)
    (1, 1, 1), (31, 2, 7), (32, 3, 8), (33, 5, 9), (127, 255, 7), (128, 256, 8), (129, 257, 9), (200, 259, 1),
    (256, 513, 9), (300, 1027, 7), (129, 3, 8), (300, 1, 9), (1, 1027, 9), (33, 257, 7),
]


@pytest.mark.parametrize("ss,dim,n", SHAPES)
def test_wmh_shapes_host_log_exact(dsk, ss, dim, n):
    rng = np.random.RandomState(ss * 7919 + dim)
    V = _weights(rng, n, dim)
    gen = dsk.WeightedMinHashGenerator(dim, ss, 13)
    par = (gen.rs, gen.ln_cs, gen.betas)
    want, _ = o.wmh_from_log(_log32(V), *par)
    assert np.array_equal(gen.minhash_batch(V), want)
    want_many, _ = o.wmh_from_log(_log32(V), *par, many=True)
    assert np.array_equal(_many_array(gen.minhash_many(V), ss), want_many)


@pytest.mark.parametrize("ss,dim,sample", [(33, 3, False), (129, 257, True), (300, 1027, True)])
def test_wmh_more_groups_than_ctas(dsk, ss, dim, sample):
    """n = 2 * 8 * 8 * sm_count + 3: each CTA of the capped grid loops over three groups, the last one partial."""
    from datasketch_b200 import _native as nv
    n = 2 * 8 * 8 * nv.device_info(0)["sm_count"] + 3
    rng = np.random.RandomState(dim)
    V = _weights(rng, n, dim, zeros=0.5)
    gen = dsk.WeightedMinHashGenerator(dim, ss, 2)
    par = (gen.rs, gen.ln_cs, gen.betas)
    rows = np.arange(n)
    if sample:
        rows = np.unique(np.concatenate([rng.choice(n, 120, replace=False), np.arange(n - 11, n), [0, 7, 8]]))
    got = gen.minhash_batch(V)
    want, _ = o.wmh_from_log(_log32(V[rows]), *par)
    assert np.array_equal(got[rows], want)
    got = _many_array(gen.minhash_many(V), ss)
    want, _ = o.wmh_from_log(_log32(V[rows]), *par, many=True)
    assert np.array_equal(got[rows], want)


# ---- device logarithm ----------------------------------------------------------------------------------------------
def _near_midpoint(W):
    """Entries whose float64 log lies within 2 float64 ulps of a float32 rounding midpoint: there the device's
    double-then-float rounding may legitimately differ from the correctly rounded float32 log."""
    with np.errstate(divide="ignore", invalid="ignore"):
        l64 = np.log(np.asarray(W, dtype=np.float32).astype(np.float64))
    fin = np.isfinite(l64)
    l64 = np.where(fin, l64, 1.0)
    f = l64.astype(np.float32)
    other = np.nextafter(f, np.where(l64 > f.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)))
    mid = (f.astype(np.float64) + other.astype(np.float64)) / 2
    return fin & (np.abs(l64 - mid) <= 2 * np.spacing(np.abs(l64)))


def _assert_near_ties(W, par, got, want, many):
    """Every (k, t) difference between the device-log result and the numpy-log oracle is a float near-tie, confirmed
    in float64: the two columns' ln_a within a few float32 ulps, or a floor argument that close to an integer."""
    rs, ln_cs, betas = par
    with np.errstate(divide="ignore", invalid="ignore"):
        l64 = np.log(np.asarray(W, dtype=np.float32).astype(np.float64))
    bad = []
    for u, s in zip(*np.where((got != want).any(axis=2))):
        cols = np.array([got[u, s, 0], want[u, s, 0]])
        arg, ln_a = o.wmh_terms64(l64[u, cols], rs[s, cols], ln_cs[s, cols], betas[s, cols], many)
        scale_arg = np.abs(l64[u, cols] / rs[s, cols]) + betas[s, cols]
        near_int = np.abs(arg - np.round(arg)) <= 6 * np.spacing(scale_arg.astype(np.float32))
        scale = np.abs(ln_cs[s, cols]).max() + np.abs(ln_a).max() + rs[s, cols].max()
        near_tie = cols[0] != cols[1] and abs(ln_a[0] - ln_a[1]) <= 8 * np.spacing(np.float32(scale))
        if not (near_tie or near_int.any()):
            bad.append((int(u), int(s)))
    assert bad == []


@pytest.mark.parametrize("ss,dim,n", [(33, 5, 9), (129, 257, 64), (300, 1027, 16), (128, 256, 200)])
def test_wmh_device_log(dsk, ss, dim, n):
    import torch
    rng = np.random.RandomState(n + dim)
    gen = dsk.WeightedMinHashGenerator(dim, ss, 17)
    par = (gen.rs, gen.ln_cs, gen.betas)
    V = _weights(rng, n, dim)
    Vi = np.floor(_weights(rng, n, dim) * 4).astype(np.int32)
    Vi[:, 0] += 1
    V16 = _weights(rng, n, dim).clip(1e-4, 6e4).astype(np.float16)
    big = torch.from_numpy(_weights(rng, n, 2 * dim)).cuda()
    inputs = [  # (input as the user passes it, the float32 weights the kernel sees)
        (torch.from_numpy(V).cuda(), V),
        (torch.from_numpy(V.astype(np.float64) * 1.000001).cuda(), (V.astype(np.float64) * 1.000001).astype(np.float32)),
        (torch.from_numpy(V16).cuda(), V16.astype(np.float32)),
        (torch.from_numpy(Vi).cuda(), Vi.astype(np.float32)),
        (big[:, ::2], big[:, ::2].cpu().numpy()),             # non-contiguous view
        (V, V),                                              # numpy with device_log=True
    ]
    exempt = 0
    for X, W in inputs:
        near = _near_midpoint(W).any(axis=1)
        exempt += int(near.sum())
        for many in (False, True):
            if many and not isinstance(X, np.ndarray):
                got = gen._sample(X, 0, many=True)[0]
            elif many:
                got = gen._sample(X, 0, many=True, device_log=True)[0]
            else:
                got = gen.minhash_batch(X, device_log=True)
            want, _ = o.wmh_from_log(_log64to32(W), *par, many=many)
            assert np.array_equal(got[~near], want[~near]), (X.dtype, many)
            want_np, _ = o.wmh_from_log(_log32(W), *par, many=many)
            _assert_near_ties(W, par, got, want_np, many)
        if not isinstance(X, np.ndarray):
            dev = gen.minhash_batch(X, to_host=False)
            assert dev.is_cuda and dev.dtype == torch.int64
            assert np.array_equal(dev.cpu().numpy(), gen.minhash_batch(X))
    assert exempt <= 2, exempt


# ---- constructed ties and floor edges ------------------------------------------------------------------------------
TIE_PAIRS = [(0, 1), (3, 4), (255, 256), (516, 517)]   # one unroll quad, across quads, across the tile, remainder loop


@pytest.mark.parametrize("ss", [33, 130])
def test_wmh_ties_first_index(dsk, ss):
    """Column j gets column i's parameters and weight, so ln_a is equal: k = i in both modes and both log sources.
    dim 519 ends in a 7-dim tile: 516..518 run in the remainder loop."""
    import torch
    dim = 519
    gen = dsk.WeightedMinHashGenerator(dim, ss, 23)
    rs, lc, be = gen.rs.copy(), gen.ln_cs.copy(), gen.betas.copy()
    for i, j in TIE_PAIRS:
        rs[:, j], lc[:, j], be[:, j] = rs[:, i], lc[:, i], be[:, i]
    gen.rs, gen.ln_cs, gen.betas = rs, lc, be                # before the device handle is built
    rng = np.random.RandomState(ss)
    rows = []
    for i, j in TIE_PAIRS:
        v = np.zeros(dim, np.float32)
        v[i] = v[j] = rng.uniform(0.5, 5)
        rows.append(v)
    v = rng.uniform(0.1, 2, dim).astype(np.float32)
    for i, j in TIE_PAIRS:
        v[i] = v[j] = 1e4
    rows.append(v)
    v = np.zeros(dim, np.float32)
    v[-1] = 3.0                                              # only the last column of the last tile
    rows.append(v)
    V = np.stack(rows)
    for many in (False, True):
        for got, vlog in ((_raw(gen, torch.from_numpy(_log32(V)).cuda(), many | WMH_INPUT_LOG)[0], _log32(V)),
                          (_raw(gen, torch.from_numpy(V).cuda(), int(many))[0], _log64to32(V))):
            want, _ = o.wmh_from_log(vlog, rs, lc, be, many=many)
            assert np.array_equal(got, want)
            for r, (i, j) in enumerate(TIE_PAIRS):
                assert (got[r, :, 0] == i).all(), (many, i, j)
            assert not np.isin(got[len(TIE_PAIRS), :, 0], [j for _, j in TIE_PAIRS]).any()
            assert (got[-1, :, 0] == dim - 1).all()
    assert np.array_equal(gen.minhash_batch(V), o.wmh_from_log(_log32(V), rs, lc, be)[0])


def test_wmh_floor_edges(dsk):
    """vlog / r + beta an exact integer (exactly representable r and beta), and vlog one float32 ulp either side."""
    import torch
    rvals = np.array([0.5, 0.75, 1.25, 2.0, 0.375, 3.0, 1.0, 0.625], np.float32)
    bvals = np.array([0.25, 0.5, 0.125, 0.75, 0.0, 0.875, 0.5, 0.0625], np.float32)
    dim, ss = len(rvals), 130
    gen = dsk.WeightedMinHashGenerator(dim, ss, 4)
    gen.rs, gen.betas = np.tile(rvals, (ss, 1)), np.tile(bvals, (ss, 1))
    rows = []
    for m in (-40, -3, 0, 1, 4, 17, 100):
        exact = ((np.float32(m) - bvals) * rvals).astype(np.float32)
        assert np.array_equal(exact / rvals + bvals, np.full(dim, m, np.float32))
        rows += [exact, np.nextafter(exact, np.float32(np.inf)), np.nextafter(exact, np.float32(-np.inf))]
    vlog = np.stack(rows).astype(np.float32)
    par = (gen.rs, gen.ln_cs, gen.betas)
    for many in (0, WMH_MANY):
        got, st = _raw(gen, torch.from_numpy(vlog).cuda(), many | WMH_INPUT_LOG)
        want, wst = o.wmh_from_log(vlog, *par, many=bool(many))
        assert np.array_equal(st, wst) and not st.any() and np.array_equal(got, want)
        assert (want[2::3, :, 1] != want[0::3, :, 1]).any()


# ---- special weights -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["a", "b"])
def test_wmh_special_weights(dsk, golden, tag):
    """The reference's results for zeros, -0.0, negative, NaN, +-inf, subnormal and FLT_MAX weights: minhash values or
    its exception type, minhash_many values (INT64_MIN for a non-finite t) and None rows."""
    import torch
    g = golden("wmh_special")
    X = g["X"]
    dim, ss, seed = (int(x) for x in g[f"{tag}_cfg"])
    gen = dsk.WeightedMinHashGenerator(dim, ss, seed)
    err, want = g[f"{tag}_err"], g[f"{tag}_out"]
    for i, v in enumerate(X):
        if err[i]:
            with pytest.raises({"ValueError": ValueError, "OverflowError": OverflowError}[str(err[i])]):
                gen.minhash(v)
        else:
            assert np.array_equal(gen.minhash(v).hashvalues, want[i]), i
    ok = err == ""
    assert np.array_equal(gen.minhash_batch(X[ok]), want[ok])
    for bad, exc in (("ValueError", ValueError), ("OverflowError", OverflowError)):
        rows = np.where(ok | (err == bad))[0]
        with pytest.raises(exc):
            gen.minhash_batch(X[rows])
        with pytest.raises(exc):
            gen.minhash_batch(torch.from_numpy(X[rows]).cuda(), to_host=False)
    many = gen.minhash_many(X)
    null = g[f"{tag}_many_null"]
    assert [m is None for m in many] == null.tolist()
    assert all(np.array_equal(m.hashvalues, g[f"{tag}_many_out"][i]) for i, m in enumerate(many) if m is not None)
    par = (gen.rs, gen.ln_cs, gen.betas)
    for flags in (0, WMH_MANY):                               # the device logarithm on the same rows
        got, st = _raw(gen, torch.from_numpy(X).cuda(), flags)
        want_d, wst = o.wmh_from_log(_log64to32(X), *par, many=bool(flags))
        assert np.array_equal(st, wst) and np.array_equal(got, want_d)
        if flags:
            assert np.array_equal(st == 1, null) and (got[st == 2][:, :, 1] == INT64_MIN).all()
        else:
            assert np.array_equal(st == 1, err == "ValueError") and np.array_equal(st == 2, err == "OverflowError")


def test_wmh_minhash_errors_match_reference(dsk):
    gen = dsk.WeightedMinHashGenerator(6, 4, 1)
    with pytest.raises(ValueError, match="all zeros"):
        gen.minhash([0, -0.0, 0, 0, 0, 0])
    with pytest.raises(ValueError, match="All-NaN"):
        gen.minhash([-1, -2, 0, 0, 0, np.nan])
    with pytest.raises(OverflowError):
        gen.minhash([1, 2, np.inf, 4, 0, 5])
    m = gen.minhash_many(np.array([[1, 2, -3, 4, 0, 5], [-1, -2, 0, 0, 0, 0], [0] * 6], np.float32))
    assert m[2] is None and (m[0].hashvalues[:, 0] == 2).all() and (m[1].hashvalues[:, 0] == 0).all()
    assert (m[0].hashvalues[:, 1] == INT64_MIN).all() and (m[1].hashvalues[:, 1] == INT64_MIN).all()
