"""GpuLSHEnsemble's containment estimates: ``query_containment``, ``query_topk`` and ``containment_pairs``.

For query q (signature m_q, size s_q) and candidate x (a row of the ``index`` call, size s_x), with j = eq / K
(``MinHash.jaccard``), ``c = j * (s_q + s_x) / (s_q * (1 + j))`` in float64, bit for bit the Python expression over ints
and floats.  The candidates are ``query``'s; a candidate is kept iff ``c >= min_containment``; the top-k order is
``(-c, row)``; the self-join lists, for indexed row i, ``query_containment`` of row i with its own size without i.

tests/golden/lsh_ensemble_containment.npz (oracle/gen_golden_lsh_ensemble_containment.py) holds the reference's
candidates and the bits of c; the oracle here restates them with ``Oracle`` of test_lsh_ensemble_device.py.  Backends as
there: ``emu``, the library on the emulation shim through its C-ABI, and ``gpu``, the Python API on the H100.
"""
import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest

from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_lsh_ensemble_device import Oracle, _EmuEns, _GpuEns, _host, _low_entropy  # noqa: E402
from test_lsh_self_join import _aligned, _p  # noqa: E402

DSK_OK, DSK_ERR_INVALID = 0, 1


def c_ref(eq, k, sq, sx):
    """The estimate as the reference's users write it: MinHash.jaccard, then Python ints and floats."""
    j = float(eq) / float(k)
    return j * (int(sq) + int(sx)) / (int(sq) * (1 + j))


def bits(c):
    return int(np.array(c, dtype=np.float64).view(np.uint64))


# ---- backends --------------------------------------------------------------------------------------------------------------
class _EmuC(_EmuEns):
    """_EmuEns plus the containment C-ABI, with the package's min_containment check."""

    sizes = None

    def index(self, sig, sizes):
        super().index(sig, sizes)
        self.sizes = _aligned(np.asarray(sizes, dtype=np.int64))

    def _xs(self):
        return self.sizes if self.sizes is not None else _aligned(np.zeros(1, dtype=np.int64))

    def _csr(self, count, fill, items):
        lib = self.lib
        counts, iptr = np.full(items + 1, -7, dtype=np.int64), np.zeros(items + 1, dtype=np.int64)
        scratch = np.zeros(items // 1024 + 2, dtype=np.int64)
        assert count(_p(counts)) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), items, _p(iptr), _p(scratch), None) == 0
        m = int(iptr[-1])
        idx, eq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        c = np.full(max(m, 1), -7.0)
        assert fill(_p(iptr), _p(idx), _p(eq), _p(c)) == 0, lib.dsk_last_error()
        return iptr[::self.num_part], idx[:m], eq[:m], c[:m]

    def query_containment(self, qsig, qsizes, t=None):
        from datasketch_b200.lshensemble import _min_containment
        lib, t = self.lib, _min_containment(t)
        qsig = _aligned(np.asarray(qsig, dtype=np.uint32).reshape(-1, self.k))
        qs = _aligned(np.asarray(qsizes, dtype=np.int64))
        sel = _aligned(self.selection(qs).reshape(-1))
        args = (self.h, _p(qsig), len(qsig), _p(qs), _p(sel), _p(self._xs()), t)
        return self._csr(lambda cnt: lib.dsk_lsh_ensemble_containment_count(*args, cnt, None),
                         lambda ptr, idx, eq, c: lib.dsk_lsh_ensemble_containment_fill(*args, ptr, idx, eq, c, None),
                         len(qsig) * self.num_part)

    def query_topk(self, qsig, qsizes, k, t=None):
        from datasketch_b200.lshensemble import _min_containment
        lib, t = self.lib, _min_containment(t)
        qsig = _aligned(np.asarray(qsig, dtype=np.uint32).reshape(-1, self.k))
        qs = _aligned(np.asarray(qsizes, dtype=np.int64))
        sel = _aligned(self.selection(qs).reshape(-1))
        nq = len(qsig)
        idx, eq, c = np.full((nq, k), -7, dtype=np.int32), np.full((nq, k), -7, dtype=np.int32), np.full((nq, k), -7.0)
        rc = lib.dsk_lsh_ensemble_containment_topk(self.h, _p(qsig), nq, _p(qs), _p(sel), _p(self._xs()), t, k, _p(idx),
                                                   _p(eq), _p(c), None)
        assert rc == 0, lib.dsk_last_error()
        return idx, eq, c

    def containment_pairs(self, t=None):
        from datasketch_b200.lshensemble import _min_containment
        lib, t = self.lib, _min_containment(t)
        if self.sizes is None:
            return np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32), np.zeros(0, dtype=np.int32), np.zeros(0)
        sel = _aligned(self.selection(self.sizes).reshape(-1))
        args = (self.h, _p(sel), _p(self.sizes), t)
        return self._csr(lambda cnt: lib.dsk_lsh_ensemble_self_containment_count(*args, cnt, None),
                         lambda ptr, idx, eq, c: lib.dsk_lsh_ensemble_self_containment_fill(*args, ptr, idx, eq, c, None),
                         len(self.sizes) * self.num_part)


class _GpuC(_GpuEns):
    def query_containment(self, qsig, qsizes, t=None):
        return self.ix.query_containment(np.ascontiguousarray(qsig, dtype=np.uint32), np.asarray(qsizes, dtype=np.int64), t)

    def query_topk(self, qsig, qsizes, k, t=None):
        return self.ix.query_topk(np.ascontiguousarray(qsig, dtype=np.uint32), np.asarray(qsizes, dtype=np.int64), k, t)

    def containment_pairs(self, t=None):
        return self.ix.containment_pairs(t)


class _Emu:
    name = "emu"
    grid_items = 2 * 8 * 8

    def __init__(self, lib):
        self.lib = lib

    def ensemble(self, thr, k, num_part, m):
        return _EmuC(self.lib, thr, k, num_part, m)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.grid_items = dsk._native.device_info(0)["sm_count"] * 8 * 8

    def ensemble(self, thr, k, num_part, m):
        return _GpuC(thr, k, num_part, m)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


# ---- expected results ------------------------------------------------------------------------------------------------------
def _lists(ptr, idx, eq, c):
    """Per query {row: (eq, bits of c)}; each row once."""
    assert ptr[0] == 0 and np.all(np.diff(ptr) >= 0) and ptr[-1] == len(idx) == len(eq) == len(c)
    cb = np.asarray(c, dtype=np.float64).view(np.uint64)
    out = []
    for q in range(len(ptr) - 1):
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        d = dict(zip(idx[sl].tolist(), zip(eq[sl].tolist(), cb[sl].tolist())))
        assert len(d) == sl.stop - sl.start, q
        out.append(d)
    return out


def _cut(want, t):
    """want filtered at min_containment t (None keeps all)."""
    if t is None:
        return want
    return [{x: v for x, v in w.items() if np.uint64(v[1]).view(np.float64) >= t} for w in want]


def _topk(want, k, t=None):
    """(idx, eq, bits) [Q, k] of the kept candidates in the order (-c, row), padded with -1 / -1 / -1.0."""
    nq = len(want)
    idx, eq = np.full((nq, k), -1, dtype=np.int32), np.full((nq, k), -1, dtype=np.int32)
    cb = np.full((nq, k), bits(-1.0), dtype=np.uint64)
    for q, w in enumerate(_cut(want, t)):
        order = sorted(w.items(), key=lambda kv: (-float(np.uint64(kv[1][1]).view(np.float64)), kv[0]))[:k]
        for j, (x, (e, b)) in enumerate(order):
            idx[q, j], eq[q, j], cb[q, j] = x, e, b
    return idx, eq, cb


def _check_topk(got, want, k, t=None):
    gi, ge, gc = (np.asarray(x) for x in got)
    wi, we, wc = _topk(want, k, t)
    assert gi.shape == wi.shape
    assert np.array_equal(gi, wi) and np.array_equal(ge, we)
    assert np.array_equal(np.ascontiguousarray(gc, dtype=np.float64).view(np.uint64), wc)


def _want_oracle(host, sig, sizes, qsig, qsizes, self_join=False):
    """Oracle restatement: candidates of test_lsh_ensemble_device's Oracle, eq by numpy, c by c_ref."""
    orc = Oracle(host, sig, [int(s) for s in sizes])
    k = host.h
    sig = np.asarray(sig, dtype=np.uint32)
    out = []
    for i, (q, s) in enumerate(zip(np.asarray(qsig, dtype=np.uint32), qsizes)):
        xs = orc.query(q, int(s)) - ({i} if self_join else set())
        out.append({x: (int(np.count_nonzero(q == sig[x])),
                        bits(c_ref(np.count_nonzero(q == sig[x]), k, int(s), int(sizes[x])))) for x in xs})
    return out


# ---- the fixture -----------------------------------------------------------------------------------------------------------
def _fixture_cases(golden):
    base, g = golden("lsh_ensemble"), golden("lsh_ensemble_containment")
    for c, (thr, k, num_part, m) in enumerate(g["configs"].tolist()):
        cfg = (float(thr), int(k), int(num_part), int(m))
        name = str(g["config_corpus"][c])
        sigs = []
        for which in ("", "q"):
            ptr, tok = base[name + "_" + which + "tok_ptr"], base[name + "_" + which + "tok"].astype(np.uint64)
            sig = o.bulk_signatures_csr(tok, ptr, cfg[1], 1).astype(np.uint32)
            assert hashlib.sha256(sig.astype("<u4").tobytes()).hexdigest() == str(g["c%d_%ssig_sha256" % (c, which)])
            sigs.append(sig)
        want = {}
        for key in ("q", "s"):
            ptr = g["c%d_%s_ptr" % (c, key)]
            want[key] = _lists(ptr, g["c%d_%s_idx" % (c, key)], g["c%d_%s_eq" % (c, key)],
                               g["c%d_%s_cbits" % (c, key)].view(np.float64))
        yield c, cfg, sigs[0], g["c%d_sizes" % c], sigs[1], g["c%d_qsizes" % c], want, g


def test_oracle_restates_the_fixture(golden):
    """The oracle's candidates, eq and bits of c are the reference's, for every configuration: K = 128, 64 (40
    partitions, trailing None uppers), 100 and 320, and sizes times 10^13 where s_q + s_x exceeds 2^53.  The fixture
    has estimates above 1, and the integer form eq*(s_q+s_x) / (s_q*(K+eq)) differs from it in the last bit somewhere."""
    seen_big = seen_over1 = seen_none = False
    int_form_differs = 0
    for c, cfg, sig, sizes, qsig, qsizes, want, g in _fixture_cases(golden):
        host = _host(*cfg)
        assert _want_oracle(host, sig, sizes, qsig, qsizes) == want["q"], c
        assert _want_oracle(host, sig, sizes, sig, sizes, self_join=True) == want["s"], c
        orc = Oracle(host, sig, [int(s) for s in sizes])
        assert [-1 if x is None else int(x) for x in orc.uppers] == g["c%d_uppers" % c].tolist()
        seen_none |= orc.uppers[-1] is None
        seen_big |= int(sizes.max()) + int(qsizes.max()) > 2 ** 53
        for w, ss in ((want["q"], qsizes), (want["s"], sizes)):
            for q, d in enumerate(w):
                for x, (e, b) in d.items():
                    cv = float(np.uint64(b).view(np.float64))
                    seen_over1 |= cv > 1.0
                    int_form_differs += (e * (int(ss[q]) + int(sizes[x]))) / (int(ss[q]) * (cfg[1] + e)) != cv
    assert seen_big and seen_over1 and seen_none and int_form_differs > 0


def test_fixture(be, golden):
    """Every configuration of the fixture: the candidates with eq and the bits of c, filtered at None, 0, the ensemble's
    threshold, 1.0, exactly at a stored c (kept) and at the next float above it (dropped); the top-k at k = 1, 5, 32;
    the self-join at None and 0.8."""
    for c, cfg, sig, sizes, qsig, qsizes, want, _ in _fixture_cases(golden):
        ens = be.ensemble(*cfg)
        try:
            ens.index(sig, sizes)
            wq = want["q"]
            vals = sorted(float(np.uint64(b).view(np.float64)) for d in wq for _, b in d.values())
            at = [v for v in vals if 0.0 < v < 1.0][len(vals) // 3]
            for t in (None, 0.0, cfg[0], 1.0, at, float(np.nextafter(at, 2.0))):
                assert _lists(*ens.query_containment(qsig, qsizes, t)) == _cut(wq, t), (c, t)
            assert any(at in [float(np.uint64(b).view(np.float64)) for _, b in d.values()] for d in _cut(wq, at))
            for k in (1, 5, 32):
                _check_topk(ens.query_topk(qsig, qsizes, k), wq, k)
            _check_topk(ens.query_topk(qsig, qsizes, 5, cfg[0]), wq, 5, cfg[0])
            for t in (None, 0.8):
                assert _lists(*ens.containment_pairs(t)) == _cut(want["s"], t), (c, t)
        finally:
            ens.close()


# ---- consistency, order and ties ---------------------------------------------------------------------------------------------
def _corpus(rs, n, k, nq, vals=3):
    sig = _low_entropy(rs, n, k, vals)
    sig[:, 12:] = rs.randint(0, 1 << 32, size=(n, k - 12), dtype=np.uint64).astype(np.uint32)
    sig[n // 2:, 12:] = sig[rs.randint(0, n // 2, n - n // 2), 12:]        # near-duplicates: large eq
    sizes = np.clip((rs.pareto(1.0, n) * 20 + 1).astype(np.int64), 1, 5000)
    qsig = sig[rs.randint(0, n, nq)].copy()
    qsig[:, 12 + k // 4:] = rs.randint(0, 1 << 32, size=(nq, k - 12 - k // 4), dtype=np.uint64)
    qsizes = rs.randint(1, 3000, nq)
    return sig, sizes, qsig, qsizes


def test_consistency_with_query_and_each_other(be):
    """query_containment(None) is query(with_eq=True) with c; query_topk is the first k of query_containment sorted by
    (-c, row); containment_pairs is query_containment of each indexed row with its own size, without itself."""
    rs = np.random.RandomState(11)
    n, nq = (150, 40) if be.name == "emu" else (3000, 500)
    sig, sizes, qsig, qsizes = _corpus(rs, n, 64, nq)
    ens = be.ensemble(0.5, 64, 8, 4)
    try:
        ens.index(sig, sizes)
        full = _lists(*ens.query_containment(qsig, qsizes))
        ptr, idx, eq = ens.query(qsig, qsizes, with_eq=True)
        assert [{x: v[0] for x, v in d.items()} for d in full] == \
            [dict(zip(idx[ptr[q]:ptr[q + 1]].tolist(), eq[ptr[q]:ptr[q + 1]].tolist())) for q in range(nq)]
        assert all(v[1] == bits(c_ref(v[0], 64, qsizes[q], sizes[x])) for q, d in enumerate(full) for x, v in d.items())
        assert sum(len(d) for d in full) > nq and max(len(d) for d in full) > 5
        for k, t in ((1, None), (5, None), (5, 0.5), (32, 0.3)):
            _check_topk(ens.query_topk(qsig, qsizes, k, t), full, k, t)
        own = _lists(*ens.query_containment(sig, sizes))
        for i, d in enumerate(own):
            d.pop(i, None)
        pairs = _lists(*ens.containment_pairs())
        assert pairs == own and sum(len(d) for d in pairs) > n // 2
        assert _lists(*ens.containment_pairs(0.6)) == _cut(own, 0.6)
    finally:
        ens.close()


def _equal_c_groups(k, sq, sizes):
    """Groups of (eq, s_x) pairs, eq >= 4, with bit-equal c for query size sq; searched, not assumed."""
    groups = {}
    for e in range(4, k + 1):
        for sx in sizes:
            groups.setdefault(bits(c_ref(e, k, sq, sx)), []).append((e, sx))
    return [v for v in groups.values() if len({e for e, _ in v}) >= 2]


def test_order_and_ties(be):
    """Rows shuffled so set numbers differ from rows (a tie-break on the set number fails); identical rows with equal
    sizes (both listed, ordered by row); equal c from different (eq, s_x) pairs; buckets with more candidates than k,
    fewer (padding), and k = 1.  Every candidate shares band 0 with its query (eq >= 4 leading positions)."""
    k, sq = 32, 12
    rs = np.random.RandomState(12)
    size_pool = list(range(2, 40))
    groups = _equal_c_groups(k, sq, size_pool)
    assert groups
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
    rows, sizes = [], []

    def add(e, sx, copies=1):
        r = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
        r[:e] = q[:e]
        for _ in range(copies):
            rows.append(r.copy())
            sizes.append(sx)
    for g in groups[:4]:
        for e, sx in g[:3]:
            add(e, sx)
    add(20, 15, copies=3)                                                  # identical rows, equal sizes
    for e in rs.randint(4, k + 1, 12).tolist():
        add(e, int(rs.choice(size_pool)))
    copies = [len(rows) - 3 - 12 + i for i in range(3)]
    rows, sizes = np.stack(rows), np.array(sizes, dtype=np.int64)
    perm = rs.permutation(len(rows))
    rows, sizes = rows[perm], sizes[perm]
    copies = [int(np.flatnonzero(perm == c)[0]) for c in copies]           # the copies' rows after the shuffle
    assert len(rows) < 32
    qsig = np.stack([q, rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)])   # the second: no candidate
    qs = np.array([sq, sq])
    ens = be.ensemble(0.5, k, 1, 4)
    try:
        ens.index(rows, sizes)
        full = _lists(*ens.query_containment(qsig, qs))
        assert len(full[0]) == len(rows) and len(full[1]) == 0
        cs = [v[1] for v in full[0].values()]
        assert len(cs) - len(set(cs)) >= 4                                 # ties in c
        for kk in (1, 5, 32):                                              # more candidates than k, and fewer (padding)
            _check_topk(ens.query_topk(qsig, qs, kk), full, kk)
        pairs = _lists(*ens.containment_pairs())
        for i in copies:                                                   # each copy lists the other two, not itself
            assert set(copies) - {i} <= set(pairs[i]) and i not in pairs[i]
            assert pairs[i][copies[0] if i != copies[0] else copies[1]][1] == bits(1.0)
    finally:
        ens.close()


def test_extreme_sizes_and_estimates_above_one(be):
    """s_x < s_q and s_x > s_q with c > 1, unclamped; sizes 1 and 2^62 - 1 on both sides."""
    k = 32
    rs = np.random.RandomState(13)
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
    rows = np.stack([q.copy() for _ in range(6)])
    for i, e in enumerate([32, 30, 20, 8, 31, 16]):
        rows[i, e:] = ~q[e:]
    top = (1 << 62) - 1
    sizes = np.array([1, 10, 1000, top, top - 12345, 7], dtype=np.int64)
    qs = np.array([1, 10, top, 3 * 10 ** 17], dtype=np.int64)
    qsig = np.stack([q] * 4)
    ens = be.ensemble(0.5, k, 1, 4)
    try:
        ens.index(rows, sizes)
        got = _lists(*ens.query_containment(qsig, qs))
        want = [{x: (int(np.count_nonzero(q == rows[x])), bits(c_ref(np.count_nonzero(q == rows[x]), k, s, sizes[x])))
                 for x in range(6) if np.count_nonzero(q[:4] == rows[x, :4]) == 4} for s in qs.tolist()]
        assert got == want
        cvals = [float(np.uint64(v[1]).view(np.float64)) for d in got for v in d.values()]
        assert max(cvals) > 1e15 and min(cvals) < 1.0                   # unclamped above 1, and below 1
        _check_topk(ens.query_topk(qsig, qs, 3, 0.5), want, 3, 0.5)
        pairs = _lists(*ens.containment_pairs())
        assert pairs == _want_oracle(ens.host, rows, sizes, rows, sizes, self_join=True)
    finally:
        ens.close()


def test_one_set_no_queries_never_built_and_grid_sweep(be):
    k = 32
    ens = be.ensemble(0.5, k, 4, 4)
    row = np.arange(k, dtype=np.uint32)[None]
    try:
        ptr, idx, eq, c = ens.query_containment(row, [5])                   # never built
        assert ptr.tolist() == [0, 0] and len(idx) == len(eq) == len(c) == 0
        ti, te, tc = ens.query_topk(row, [5], 3)
        assert np.asarray(ti).tolist() == [[-1] * 3] and np.asarray(te).tolist() == [[-1] * 3]
        assert np.asarray(tc).tolist() == [[-1.0] * 3]
        assert [len(x) for x in ens.containment_pairs()] == [1, 0, 0, 0]
        ens.index(row, [7])
        assert _lists(*ens.query_containment(np.concatenate([row, row]), [7, 14])) == \
            [{0: (k, bits(1.0))}, {0: (k, bits(c_ref(k, k, 14, 7)))}]
        ptr, idx, eq, c = ens.query_containment(np.zeros((0, k), dtype=np.uint32), np.zeros(0, dtype=np.int64))
        assert np.asarray(ptr).tolist() == [0] and len(idx) == 0
        assert np.asarray(ens.query_topk(np.zeros((0, k), dtype=np.uint32), np.zeros(0, dtype=np.int64), 4)[0]).shape == (0, 4)
        pairs = ens.containment_pairs()
        assert np.asarray(pairs[0]).tolist() == [0, 0] and len(pairs[1]) == 0
    finally:
        ens.close()
    rs = np.random.RandomState(14)
    n = 200 if be.name == "emu" else 500                                   # every row is a candidate of every query
    sig = _low_entropy(rs, n, k, 3)
    sizes = rs.randint(1, 400, n)
    nq = (3 * be.grid_items) // 8 + 5                                      # items and queries beyond one grid sweep
    qsig, qsizes = sig[rs.randint(0, n, nq)], rs.randint(1, 400, nq)
    ens = be.ensemble(0.4, k, 8, 4)
    try:
        ens.index(sig, sizes)
        assert nq * 8 > be.grid_items and nq > be.grid_items // 8
        want = _want_oracle(ens.host, sig, sizes, qsig, qsizes)
        assert _lists(*ens.query_containment(qsig, qsizes, 0.3)) == _cut(want, 0.3)
        _check_topk(ens.query_topk(qsig, qsizes, 4), want, 4)
        assert _lists(*ens.containment_pairs(0.3)) == _cut(_want_oracle(ens.host, sig, sizes, sig, sizes, True), 0.3)
    finally:
        ens.close()


# ---- errors ----------------------------------------------------------------------------------------------------------------
def test_c_abi_argument_validation(emu_lib):
    lib, k = emu_lib, 32
    buf = _aligned(np.zeros(256, dtype=np.int64))
    b, r = np.array([4, 8], dtype=np.int32), np.array([2, 4], dtype=np.int32)
    h = ctypes.c_void_p()
    assert lib.dsk_lsh_ensemble_create(k, 2, _p(b), _p(r), 2, 0, ctypes.byref(h)) == DSK_OK
    P = _p(buf)
    try:
        # never built: the self-join is a no-op even with null buffers, the query count writes zeros
        assert lib.dsk_lsh_ensemble_self_containment_count(h, None, None, 0.5, None, None) == DSK_OK
        assert lib.dsk_lsh_ensemble_self_containment_fill(h, None, None, 0.5, None, None, None, None, None) == DSK_OK
        cnt = _aligned(np.full(2, -7, dtype=np.int64))
        assert lib.dsk_lsh_ensemble_containment_count(h, P, 1, P, P, P, 0.5, _p(cnt), None) == DSK_OK
        assert cnt.tolist() == [0, 0]
        sig = _aligned(np.arange(10 * k, dtype=np.uint32).reshape(10, k) % 3)
        order = _aligned(np.arange(10, dtype=np.int32))
        st = np.array([0, 5, 10], dtype=np.int64)
        assert lib.dsk_lsh_ensemble_index(h, _p(sig), 10, _p(order), _p(st), None) == DSK_OK
        calls = {
            "count": (lib.dsk_lsh_ensemble_containment_count, lambda hh, nq, t, bufs: (hh, bufs[0], nq, bufs[1], bufs[2], bufs[3], t, bufs[4], None), 5),
            "fill": (lib.dsk_lsh_ensemble_containment_fill, lambda hh, nq, t, bufs: (hh, bufs[0], nq, bufs[1], bufs[2], bufs[3], t, *bufs[4:], None), 8),
            "topk": (lib.dsk_lsh_ensemble_containment_topk, lambda hh, nq, t, bufs: (hh, bufs[0], nq, bufs[1], bufs[2], bufs[3], t, 4, *bufs[4:], None), 7),
        }
        for name, (fn, mk, nb) in calls.items():
            good = [P] * nb
            assert fn(*mk(None, 1, 0.5, good)) == DSK_ERR_INVALID and b"null handle" in lib.dsk_last_error()
            assert fn(*mk(h, -1, 0.5, good)) == DSK_ERR_INVALID and b"nq must be" in lib.dsk_last_error()
            for j in range(nb):
                bad = list(good)
                bad[j] = None
                assert fn(*mk(h, 1, 0.5, bad)) == DSK_ERR_INVALID and b"null buffer" in lib.dsk_last_error(), (name, j)
            for t in (float("nan"), -0.01, 1.01, float("inf")):
                assert fn(*mk(h, 1, t, good)) == DSK_ERR_INVALID and b"min_containment" in lib.dsk_last_error()
            assert fn(*mk(h, 0, 0.5, [None] * nb)) == DSK_OK
        for kk in (0, 33):
            assert lib.dsk_lsh_ensemble_containment_topk(h, P, 1, P, P, P, 0.5, kk, P, P, P, None) == DSK_ERR_INVALID
            assert b"k must be" in lib.dsk_last_error()
        assert lib.dsk_lsh_ensemble_self_containment_count(None, P, P, 0.5, P, None) == DSK_ERR_INVALID
        for args in ((None, P, 0.5, P), (P, None, 0.5, P), (P, P, 0.5, None)):
            assert lib.dsk_lsh_ensemble_self_containment_count(h, *args, None) == DSK_ERR_INVALID
        for j in range(6):
            bad = [P] * 6
            bad[j] = None
            assert lib.dsk_lsh_ensemble_self_containment_fill(h, bad[0], bad[1], 0.5, *bad[2:], None) == DSK_ERR_INVALID
        for t in (float("nan"), 2.0):
            assert lib.dsk_lsh_ensemble_self_containment_fill(h, P, P, t, P, P, P, P, None) == DSK_ERR_INVALID
            assert lib.dsk_lsh_ensemble_self_containment_count(h, P, P, t, P, None) == DSK_ERR_INVALID
    finally:
        lib.dsk_lsh_ensemble_destroy(h)


def test_min_containment_argument():
    from datasketch_b200.lshensemble import _min_containment
    assert _min_containment(None) == 0.0 and _min_containment(1) == 1.0 and _min_containment(np.float32(0.5)) == 0.5
    for bad in (float("nan"), -0.1, 1.0000001, "0.5", True, [0.5]):
        with pytest.raises(ValueError):
            _min_containment(bad)


# ---- GPU only --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_errors_and_tensor_outputs():
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(15)
    k = 64
    sig, sizes, qsig, qsizes = _corpus(rs, 400, k, 30)
    ens = dsk.GpuLSHEnsemble(threshold=0.5, num_perm=k, num_part=8, m=4)
    ens.index(sig, sizes)
    for bad in (np.zeros(30, dtype=np.int64), np.full(30, 1 << 62, dtype=np.int64), -qsizes):
        with pytest.raises(ValueError):
            ens.query_containment(qsig, bad)
        with pytest.raises(ValueError):
            ens.query_topk(qsig, bad, 3)
    for t in (float("nan"), -0.5, 1.5):
        with pytest.raises(ValueError):
            ens.query_containment(qsig, qsizes, t)
        with pytest.raises(ValueError):
            ens.query_topk(qsig, qsizes, 3, t)
        with pytest.raises(ValueError):
            ens.containment_pairs(t)
    for kk in (0, 33):
        with pytest.raises(ValueError):
            ens.query_topk(qsig, qsizes, kk)
    with pytest.raises(ValueError, match="Expecting minhash with length"):
        ens.query_containment(qsig[:, :k - 1], qsizes)
    with pytest.raises(TypeError):
        ens.query_topk(torch.zeros((2, k), dtype=torch.int64, device="cuda"), [1, 1], 2)
    host = _lists(*ens.query_containment(qsig, qsizes, 0.2))
    d_q = torch.from_numpy(qsig.view(np.int32)).cuda()
    out = ens.query_containment(d_q, qsizes, 0.2, to_host=False)
    assert all(x.is_cuda for x in out) and [x.dtype for x in out] == [torch.int64, torch.int32, torch.int32, torch.float64]
    assert _lists(*(x.cpu().numpy() for x in out)) == host
    tk = ens.query_topk(d_q, qsizes, 6, to_host=False)
    assert all(x.is_cuda for x in tk) and [x.dtype for x in tk] == [torch.int32, torch.int32, torch.float64]
    assert tk[0].shape == (30, 6)
    pr = ens.containment_pairs(0.5, to_host=False)
    assert all(x.is_cuda for x in pr) and pr[0].shape == (401,)


@pytest.mark.gpu
def test_scale_one_million_sets():
    """1M sets (K = 128, 0.5 / 16 partitions / m = 8) and 10k queries: a sample of query_containment(0.8) against c
    computed in torch from query(with_eq=True) and the sizes, query_topk(10) against the sorted lists, and
    containment_pairs(0.8) against query_containment(0.8) of the same rows with their own sizes, in chunks."""
    import torch
    import datasketch_b200 as dsk
    n, k, nq = 1_000_000, 128, 10_000
    g = torch.Generator(device="cuda").manual_seed(5)
    sig = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, k), dtype=torch.int32, device="cuda", generator=g)
    half = n // 2
    src = torch.randint(0, half, (n - half,), device="cuda", generator=g)
    sig[half:, :96] = sig[src, :96]                                       # near-duplicates: c around 0.8
    rs = np.random.RandomState(5)
    sizes = np.clip((rs.pareto(1.2, n) * 50 + 10).astype(np.int64), 10, 100_000)
    mag = 10 ** np.maximum(np.floor(np.log10(sizes)).astype(np.int64) - 1, 0)
    sizes = sizes // mag * mag
    qsig = sig[torch.randint(0, n, (nq,), device="cuda", generator=g)].clone()
    qsizes = np.clip((rs.pareto(1.2, nq) * 50 + 1).astype(np.int64), 1, 10 ** 6)
    ens = dsk.GpuLSHEnsemble(threshold=0.5, num_perm=k, num_part=16, m=8)
    ens.index(sig, sizes)
    ptr, idx, eq = ens.query(qsig, qsizes, with_eq=True, to_host=False)
    d_sz = torch.from_numpy(sizes).cuda()
    sq = torch.repeat_interleave(torch.from_numpy(qsizes).cuda(), ptr.diff())
    j = eq.double() / k
    c = j * (sq + d_sz[idx.long()]).double() / (sq.double() * (1 + j))
    keep = c >= 0.8
    cptr, cidx, ceq, cc = ens.query_containment(qsig, qsizes, 0.8)
    assert cptr[-1] == int(keep.sum()) and cptr[-1] > 1000
    ptr_h, idx_h, eq_h, c_h, keep_h = (x.cpu().numpy() for x in (ptr, idx, eq, c, keep))
    ti, te, tc = ens.query_topk(qsig, qsizes, 10, 0.8)
    for q in np.random.RandomState(2).choice(nq, 300, replace=False).tolist():
        sl = slice(int(ptr_h[q]), int(ptr_h[q + 1]))
        want = {x: (e, bits(v)) for x, e, v, kp in zip(idx_h[sl].tolist(), eq_h[sl].tolist(), c_h[sl].tolist(),
                                                      keep_h[sl].tolist()) if kp}
        assert _lists(cptr[q:q + 2] - cptr[q], cidx[cptr[q]:cptr[q + 1]], ceq[cptr[q]:cptr[q + 1]],
                      cc[cptr[q]:cptr[q + 1]]) == [want], q
        wi, we, wc = _topk([want], 10)
        assert np.array_equal(ti[q], wi[0]) and np.array_equal(te[q], we[0]) and np.array_equal(tc[q].view(np.uint64), wc[0])
    pptr, pidx, peq, pc = ens.containment_pairs(0.8)
    assert len(pptr) == n + 1 and pptr[-1] > 1000
    chunk = 100_000
    for lo in range(0, n, chunk):
        qp, qi, qe, qc = ens.query_containment(sig[lo:lo + chunk], sizes[lo:lo + chunk], 0.8)
        rows = np.repeat(np.arange(lo, lo + len(qp) - 1), np.diff(qp))
        notself = qi != rows
        sl = slice(int(pptr[lo]), int(pptr[lo + len(qp) - 1]))
        prow = np.repeat(np.arange(lo, lo + len(qp) - 1), np.diff(pptr[lo:lo + len(qp)]))
        a = np.lexsort((qi[notself], rows[notself]))
        b = np.lexsort((pidx[sl], prow))
        assert np.array_equal(rows[notself][a], prow[b]) and np.array_equal(qi[notself][a], pidx[sl][b])
        assert np.array_equal(qe[notself][a], peq[sl][b])
        assert np.array_equal(qc[notself][a].view(np.uint64), pc[sl][b].view(np.uint64))
