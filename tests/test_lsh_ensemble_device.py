"""GpuLSHEnsemble: MinHashLSHEnsemble's containment search (lshensemble.py:189-249) on the device.

``query(sig, sizes)`` lists, per query row, the rows of the ``index`` call that the reference's ``query(m, size)`` yields:
over every partition p with an upper bound, with ``(b, r) = params[searchsorted(xqs, upper_p / size)]`` (clamped), the
sets of p that share the query's r-tuple in one of the first b bands of the ``(K // r, r)`` banding.  ``eq`` is the number
of the K positions where the two rows agree.

The oracle restates the ensemble over ``oracle_np``'s dict buckets: the reference's partition walk, one first-b-bands
dict index per partition and r.  tests/golden/lsh_ensemble.npz (oracle/gen_golden_lsh_ensemble.py) pins it to the
reference.  The two backends are those of test_lsh_query_jaccard.py: ``emu``, the whole library on the emulation shim
driven through its C-ABI (with the package's own host-side planning), and ``gpu``, the Python API on the H100.
"""
import ctypes
import hashlib
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

from oracle import oracle_np as o

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_model as hm  # noqa: E402
from test_lsh_self_join import _aligned, _p  # noqa: E402

DSK_OK, DSK_ERR_INVALID = 0, 1

_HOST = {}


def _host(thr, k, num_part, m):
    """The host class of a configuration: its params / xqs / _get_optimal_param (computed once per configuration)."""
    from datasketch_b200.lshensemble import MinHashLSHEnsemble
    key = (thr, k, num_part, m)
    if key not in _HOST:
        _HOST[key] = MinHashLSHEnsemble(threshold=thr, num_perm=k, num_part=num_part, m=m)
    return _HOST[key]


# ---- the ensemble model: fingerprint seeded with the partition --------------------------------------------------------
def ens_seed(band, part):
    """The value band_fp's seed is xored with in the ensemble's tables: the band, and the partition in the high word."""
    return int(band) | (int(part) << 32)


def ens_fp(tuples, band, part):
    return hm.tuple_fp(tuples, np.uint64(ens_seed(band, part)))


# ---- oracle ------------------------------------------------------------------------------------------------------------
class Oracle:
    """MinHashLSHEnsemble over dict buckets: the reference's partition walk over the size-sorted sets (one step on when
    a size exceeds the current upper bound), per partition and r a DictLSH-style table list, queried over its first b
    bands.  Keys are the rows of the indexed matrix."""

    def __init__(self, host, sig, sizes):
        from datasketch_b200.lshensemble import optimal_partitions
        from collections import Counter
        self.host, self.k = host, host.h
        num_part = len(host.indexes)
        vals, counts = np.array(sorted(Counter(int(s) for s in sizes).most_common())).T
        self.lowers, self.uppers = [None] * num_part, [None] * num_part
        for i, (lo, up) in enumerate(optimal_partitions(vals, counts, num_part)):
            self.lowers[i], self.uppers[i] = lo, up
        entries = sorted(range(len(sizes)), key=lambda j: sizes[j])
        rs = sorted({int(r) for _, r in host.params})
        self.tables = [{r: [defaultdict(set) for _ in range(self.k // r)] for r in rs} for _ in range(num_part)]
        self.part_of = np.zeros(len(sizes), dtype=np.int64)
        curr = 0
        for j in entries:
            if sizes[j] > self.uppers[curr]:
                curr += 1
            self.part_of[j] = curr
            for r, tabs in self.tables[curr].items():
                for band, (s, e) in enumerate(o.lsh_hashranges(self.k // r, r)):
                    tabs[band][o.lsh_band_key(np.asarray(sig[j], dtype=np.uint64)[s:e])].add(j)

    def params_of(self, u, size):
        b, r = self.host._get_optimal_param(u, size)
        return int(b), int(r)

    def query(self, q, size):
        q = np.asarray(q, dtype=np.uint64)
        out = set()
        for p, u in enumerate(self.uppers):
            if u is None:
                continue
            b, r = self.params_of(u, size)
            for band, (s, e) in enumerate(o.lsh_hashranges(self.k // r, r)[:b]):
                out |= self.tables[p][r][band].get(o.lsh_band_key(q[s:e]), set())
        return out


def _want(orc, sig, qsig, qsizes):
    """Per query {row: eq}."""
    sig, qsig = np.asarray(sig, dtype=np.uint32), np.asarray(qsig, dtype=np.uint32)
    return [{d: int(np.count_nonzero(q == sig[d])) for d in orc.query(q, int(s))} for q, s in zip(qsig, qsizes)]


def _got(ptr, idx, eq=None):
    assert ptr[0] == 0 and np.all(np.diff(ptr) >= 0) and ptr[-1] == len(idx)
    out = []
    for q in range(len(ptr) - 1):
        sl = slice(int(ptr[q]), int(ptr[q + 1]))
        ids = idx[sl].tolist()
        assert len(set(ids)) == len(ids), q                        # each candidate once
        out.append(dict(zip(ids, eq[sl].tolist() if eq is not None else [None] * len(ids))))
    return out


# ---- backends ----------------------------------------------------------------------------------------------------------
class _EmuEns:
    """The emulated library through its C-ABI, with the package's host-side planning (_index_plan, _selection)."""

    def __init__(self, lib, thr, k, num_part, m):
        self.lib, self.k, self.num_part = lib, k, num_part
        self.host = _host(thr, k, num_part, m)
        self.params, self.xqs = self.host.params, self.host.xqs
        b = np.ascontiguousarray(self.params[:, 0], dtype=np.int32)
        r = np.ascontiguousarray(self.params[:, 1], dtype=np.int32)
        self.h = ctypes.c_void_p()
        assert lib.dsk_lsh_ensemble_create(k, num_part, _p(b), _p(r), len(b), 0, ctypes.byref(self.h)) == 0, \
            lib.dsk_last_error()
        self.uppers, self.start = [None] * num_part, np.zeros(num_part + 1, dtype=np.int64)

    def index(self, sig, sizes):
        from datasketch_b200.lshensemble import _index_plan
        sig = _aligned(np.asarray(sig, dtype=np.uint32))
        sizes = np.asarray(sizes, dtype=np.int64)
        self.lowers, self.uppers, order, self.start = _index_plan(sizes, self.num_part)
        order = _aligned(order.astype(np.int32))
        rc = self.lib.dsk_lsh_ensemble_index(self.h, _p(sig), len(sig), _p(order), _p(self.start), None)
        assert rc == 0, self.lib.dsk_last_error()

    def selection(self, sizes):
        from datasketch_b200.lshensemble import _selection
        return _selection(self.xqs, len(self.params), self.uppers, self.start, sizes)

    def query(self, qsig, qsizes, with_eq=True):
        lib, qsig = self.lib, _aligned(np.asarray(qsig, dtype=np.uint32).reshape(-1, self.k))
        nq = len(qsig)
        items = nq * self.num_part
        sel = _aligned(self.selection(qsizes).reshape(-1))
        counts, iptr = np.full(items + 1, -7, dtype=np.int64), np.zeros(items + 1, dtype=np.int64)
        scratch = np.zeros(items // 1024 + 2, dtype=np.int64)
        assert lib.dsk_lsh_ensemble_query_count(self.h, _p(qsig), nq, _p(sel), _p(counts), None) == 0, lib.dsk_last_error()
        assert lib.dsk_exclusive_scan(_p(counts), items, _p(iptr), _p(scratch), None) == 0
        m = int(iptr[-1])
        idx, eq = np.full(max(m, 1), -7, dtype=np.int32), np.full(max(m, 1), -7, dtype=np.int32)
        rc = lib.dsk_lsh_ensemble_query_fill(self.h, _p(qsig), nq, _p(sel), _p(iptr), _p(idx), _p(eq) if with_eq else None,
                                             None)
        assert rc == 0, lib.dsk_last_error()
        ptr = iptr[::self.num_part]
        return (ptr, idx[:m], eq[:m]) if with_eq else (ptr, idx[:m])

    def close(self):
        self.lib.dsk_lsh_ensemble_destroy(self.h)


class _GpuEns:
    def __init__(self, thr, k, num_part, m):
        import datasketch_b200 as dsk
        self.ix = dsk.GpuLSHEnsemble(threshold=thr, num_perm=k, num_part=num_part, m=m)
        self.host = _host(thr, k, num_part, m)

    def index(self, sig, sizes):
        self.ix.index(np.ascontiguousarray(sig, dtype=np.uint32), np.asarray(sizes, dtype=np.int64))
        self.lowers, self.uppers = self.ix.lowers, self.ix.uppers

    def selection(self, sizes):
        return self.ix.selection(sizes)

    def query(self, qsig, qsizes, with_eq=True):
        return self.ix.query(np.ascontiguousarray(qsig, dtype=np.uint32), np.asarray(qsizes, dtype=np.int64), with_eq=with_eq)

    def close(self):
        pass


class _Emu:
    name = "emu"
    grid_items = 2 * 8 * 8

    def __init__(self, lib):
        self.lib = lib

    def ensemble(self, thr, k, num_part, m):
        return _EmuEns(self.lib, thr, k, num_part, m)


class _Gpu:
    name = "gpu"

    def __init__(self):
        import datasketch_b200 as dsk
        self.grid_items = dsk._native.device_info(0)["sm_count"] * 8 * 8

    def ensemble(self, thr, k, num_part, m):
        return _GpuEns(thr, k, num_part, m)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


def _check(ens, sig, sizes, qsig, qsizes):
    """Index, query with and without eq, compare with the oracle (sets, eq) and the partitions; returns the oracle."""
    orc = Oracle(ens.host, sig, np.asarray(sizes).tolist())
    ens.index(sig, sizes)
    assert [None if x is None else int(x) for x in ens.uppers] == [None if x is None else int(x) for x in orc.uppers]
    want = _want(orc, sig, qsig, qsizes)
    got = _got(*ens.query(qsig, qsizes))
    assert got == want
    assert [set(g) for g in _got(*ens.query(qsig, qsizes, with_eq=False))] == [set(w) for w in want]
    return orc, want


def _low_entropy(rs, n, k, vals):
    return rs.randint(0, vals, size=(n, k)).astype(np.uint32)


def _sizes_for(host, part_upper, row):
    """A query size whose ratio part_upper / size selects row ``row`` of the (b, r) table."""
    xqs = host.xqs
    size = int(np.ceil(float(part_upper) / xqs[row]))
    assert np.searchsorted(xqs, float(part_upper) / size) == row
    return size


# ---- golden: the reference's own results ------------------------------------------------------------------------------
def _golden_corpus(g, name):
    k = {"a": 128, "b": 64, "c": 16}[name]
    out = []
    for which in ("", "q"):
        ptr, tok = g[name + "_" + which + "tok_ptr"], g[name + "_" + which + "tok"].astype(np.uint64)
        sig = o.bulk_signatures_csr(tok, ptr, k, 1).astype(np.uint32)
        assert hashlib.sha256(sig.astype("<u4").tobytes()).hexdigest() == str(g[name + "_" + which + "sig_sha256"])
        out += [sig, np.diff(ptr)]
    return out   # sig, sizes, qsig, qsizes


def _golden_cases(g):
    for c, (thr, k, num_part, m) in enumerate(g["configs"].tolist()):
        yield c, (float(thr), int(k), int(num_part), int(m)), str(g["config_corpus"][c])


def _golden_lists(g, c):
    ptr, idx = g["c%d_res_ptr" % c], g["c%d_res_idx" % c]
    return [idx[ptr[i]:ptr[i + 1]].tolist() for i in range(len(ptr) - 1)]


def test_oracle_is_the_reference(golden):
    """The oracle's partitions, per-(query, partition) (b, r) and query results are the reference's, for the four
    configurations of the fixture (default-like with r = 1 tables of 128 bands, num_part above the number of distinct
    sizes, num_part = 1, K = 16 with m = 2)."""
    g = golden("lsh_ensemble")
    seen_none = seen_r1 = False
    for c, cfg, name in _golden_cases(g):
        host = _host(*cfg)
        assert np.array_equal(host.params, g["c%d_params" % c]) and np.array_equal(host.xqs, g["c%d_xqs" % c])
        sig, sizes, qsig, qsizes = _golden_corpus(g, name)
        orc = Oracle(host, sig, sizes.tolist())
        assert [-1 if x is None else int(x) for x in orc.uppers] == g["c%d_uppers" % c].tolist()
        assert [-1 if x is None else int(x) for x in orc.lowers] == g["c%d_lowers" % c].tolist()
        for q, s in enumerate(qsizes.tolist()):
            for p, u in enumerate(orc.uppers):
                want = (0, 0) if u is None else orc.params_of(u, s)
                assert want == (int(g["c%d_b" % c][q, p]), int(g["c%d_r" % c][q, p]))
        assert [sorted(orc.query(q, int(s))) for q, s in zip(qsig, qsizes)] == _golden_lists(g, c)
        seen_none |= orc.uppers[-1] is None
        seen_r1 |= int(g["c%d_b" % c].max()) == cfg[1]
    assert seen_none and seen_r1


def test_golden(be, golden):
    """The library gives the reference's query results for every configuration of the fixture, and eq."""
    g = golden("lsh_ensemble")
    for c, cfg, name in _golden_cases(g):
        sig, sizes, qsig, qsizes = _golden_corpus(g, name)
        ens = be.ensemble(*cfg)
        try:
            _, want = _check(ens, sig, sizes, qsig, qsizes)
            got = _got(*ens.query(qsig, qsizes))
            assert [sorted(x) for x in got] == _golden_lists(g, c), c
            assert sum(len(x) for x in got) > 0
        finally:
            ens.close()


# ---- the (b, r) selection and the partition walk, on the host -----------------------------------------------------------
def test_selection_table_is_get_optimal_param(golden):
    """_selection's table row equals the host class's _get_optimal_param for every (query, partition) of the fixture and
    of a randomised sweep: sizes from 1 to 10^12, ratios on both sides of xqs[0] and xqs[-1] and exactly on the xqs
    grid's neighbours."""
    from datasketch_b200.lshensemble import _selection
    g = golden("lsh_ensemble")
    rs = np.random.RandomState(0)
    cases = []
    for c, cfg, name in _golden_cases(g):
        _, sizes, _, qsizes = _golden_corpus(g, name)
        uppers = [None if x < 0 else int(x) for x in g["c%d_uppers" % c].tolist()]
        cases.append((_host(*cfg), uppers, qsizes))
    for cfg in [(0.5, 128, 16, 8), (0.9, 64, 8, 4), (0.3, 32, 5, 2)]:
        host = _host(*cfg)
        uppers = sorted(rs.randint(1, 10 ** 6, size=cfg[2]).tolist()) + [None]
        sizes = np.concatenate([rs.randint(1, 10 ** 7, 300), [1, 2, 3, 10 ** 12],
                                [max(1, int(u / x)) for u in uppers[:3] for x in host.xqs]])
        cases.append((host, uppers, sizes))
        # ratios exactly ON the grid: xqs[i] = num / den with den a power of two, so float(num) / float(den) == xqs[i]
        # and searchsorted(side="left") gives i where side="right" would give i + 1
        ratios = [x.as_integer_ratio() for x in host.xqs.tolist()]
        assert all(float(nu) / float(de) == x for (nu, de), x in zip(ratios, host.xqs.tolist()))
        cases.append((host, [nu for nu, _ in ratios], np.array([de for _, de in ratios], dtype=np.int64)))
    for host, uppers, sizes in cases:
        start = np.arange(len(uppers) + 1)                          # every partition non-empty
        sel = _selection(host.xqs, len(host.params), uppers, start, sizes)
        for q, s in enumerate(np.asarray(sizes).tolist()):
            for p, u in enumerate(uppers):
                if u is None:
                    assert sel[q, p] == -1
                else:
                    assert tuple(host.params[sel[q, p]]) == tuple(host._get_optimal_param(u, s)), (u, s)
    assert any((sel == 0).any() for sel in [_selection(h.xqs, 10, u, np.arange(len(u) + 1), s) for h, u, s in cases])
    assert any((sel == 9).any() for sel in [_selection(h.xqs, 10, u, np.arange(len(u) + 1), s) for h, u, s in cases])


def test_partition_ranges_follow_the_reference_walk():
    """_index_plan's order is the stable size sort and its ranges are the reference's one-step walk, also where the
    back-tracking quirk makes bounds that the walk crosses in the middle of a run of equal sizes."""
    from datasketch_b200.lshensemble import _index_plan, _partition_ranges
    rs = np.random.RandomState(1)
    for t in range(60):
        n = int(rs.randint(1, 300))
        sizes = np.clip((rs.pareto(1.0, n) * 5 + 1).astype(np.int64), 1, 500) if t % 2 else rs.randint(1, 8, n)
        num_part = int(rs.randint(1, 20))
        lowers, uppers, order, start = _index_plan(sizes, num_part)
        assert np.array_equal(order, sorted(range(n), key=lambda j: sizes[j]))
        part, curr = [], 0
        for j in order:
            if sizes[j] > uppers[curr]:
                curr += 1
            part.append(curr)
        assert np.array_equal(np.repeat(np.arange(num_part), np.diff(start)), part)
    # bounds that end inside a run: the walk moves one partition per set while the size exceeds the bound
    assert _partition_ranges(np.array([1, 5, 5, 5, 5]), [1, 2, 3, 9]).tolist() == [0, 1, 2, 3, 5]


# ---- cases -------------------------------------------------------------------------------------------------------------
def test_band_limit_first_b_bands(be):
    """A set that matches the query only in a band >= b is no candidate; one that matches below and above b is listed
    once.  The query's (b, r) is a table row with b < K // r."""
    thr, k, num_part, m = 0.5, 128, 4, 8
    ens = be.ensemble(thr, k, num_part, m)
    host = ens.host
    row = next(i for i, (b, r) in enumerate(host.params.tolist()) if b < k // r and b >= 2)
    b, r = (int(x) for x in host.params[row])
    rs = np.random.RandomState(2)
    sig = rs.randint(0, 1 << 32, size=(6, k), dtype=np.uint64).astype(np.uint32)
    q = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
    sig[0, b * r:(b + 1) * r] = q[b * r:(b + 1) * r]              # band b only: absent
    sig[1, (k // r - 1) * r:(k // r) * r] = q[(k // r - 1) * r:(k // r) * r]   # last band only: absent
    sig[2, 0:r] = q[0:r]                                          # band 0 and band b: listed once
    sig[2, b * r:(b + 1) * r] = q[b * r:(b + 1) * r]
    sig[3, (b - 1) * r:b * r] = q[(b - 1) * r:b * r]              # band b - 1: present
    sizes = np.full(6, 1000)
    size = _sizes_for(host, 1000, row)
    try:
        orc, want = _check(ens, sig, sizes, q[None], [size])
        assert set(want[0]) == {2, 3}
        assert int(ens.selection([size])[0, 0]) == row
    finally:
        ens.close()


@pytest.mark.parametrize("k,m,vals", [(128, 8, 3), (320, 2, 2)])
def test_big_buckets_many_bands_and_large_k(be, k, m, vals):
    """Low-entropy rows: buckets of many sets with the same tuple, matches in several bands (listed once), the r = 1
    tables' K bands (more than 32: several lane rounds) and K = 320 (more than 256 positions)."""
    rs = np.random.RandomState(k)
    n = 120 if be.name == "emu" else 3000
    nq = 40 if be.name == "emu" else 600
    sig = _low_entropy(rs, n, k, vals)
    sig[:, vals * 7:] = rs.randint(0, 1 << 32, size=(n, k - vals * 7), dtype=np.uint64).astype(np.uint32)
    sizes = np.clip((rs.pareto(1.0, n) * 10 + 1).astype(np.int64), 1, 3000)
    qsig = np.concatenate([sig[rs.randint(0, n, nq // 2)], _low_entropy(rs, nq - nq // 2, k, vals)])
    qsig[nq // 2:, vals * 7:] = rs.randint(0, 1 << 32, size=(nq - nq // 2, k - vals * 7), dtype=np.uint64)
    qsizes = np.concatenate([[1, 10 ** 9], rs.randint(1, 5000, nq - 2)])
    ens = be.ensemble(0.5, k, 8, m)
    try:
        _, want = _check(ens, sig, sizes, qsig, qsizes)
        assert max(len(w) for w in want) >= 10
        assert int(ens.host.params[:, 1].min()) == 1 and ens.selection(qsizes).max() >= 0
    finally:
        ens.close()


def test_equal_sizes_at_partition_boundaries_and_input_rows(be):
    """Many sets of equal size on both sides of partition bounds, rows given in shuffled order: the stable size order
    decides the partition of each set, and the results are rows of the index call (not size-order numbers)."""
    k = 32
    rs = np.random.RandomState(5)
    n = 150 if be.name == "emu" else 2000
    sizes = rs.choice([3, 3, 3, 7, 7, 8, 20, 20, 20, 21, 50], size=n)
    sig = _low_entropy(rs, n, k, 2)
    sig[:, 8:] = rs.randint(0, 1 << 32, size=(n, k - 8), dtype=np.uint64).astype(np.uint32)
    qsig = sig[rs.randint(0, n, 40)]
    qsizes = rs.choice([1, 3, 7, 20, 100], size=40)
    ens = be.ensemble(0.5, k, 4, 4)
    try:
        orc, want = _check(ens, sig, sizes, qsig, qsizes)
        assert len(set(orc.part_of.tolist())) >= 3
        assert any(len(w) > 0 for w in want)
    finally:
        ens.close()


@pytest.mark.parametrize("head_collides", [False, True])
def test_fingerprint_collisions_inside_and_across_partitions(be, head_collides):
    """Tuples with equal partition-keyed fingerprints that are not equal (hash_model second preimages under the new
    seeding): inside one partition, and across two partitions in the same band (a tuple of partition 1 built to reach the
    fingerprint of partition 0's tuple); plus the tuple whose fingerprint is the tables' empty key.  A query carrying one
    tuple meets the colliding members in its chain and must skip them.  The colliding members are inserted last or first
    (set numbers follow the size order), so the chain's head is one of them in one of the two runs."""
    thr, k, num_part, m = 0.5, 16, 2, 2
    ens = be.ensemble(thr, k, num_part, m)
    host = ens.host
    row = next(i for i, (b, r) in enumerate(host.params.tolist()) if r == 2 and b >= 2)
    b, r = (int(x) for x in host.params[row])
    rs = np.random.RandomState(40 + head_collides)
    s0, s1 = 100, 101                                              # two distinct sizes: partitions (100, 100), (101, 101)
    base = rs.randint(0, 1 << 32, size=(20, k), dtype=np.uint64).astype(np.uint32)
    band = 1
    sl = slice(band * r, (band + 1) * r)
    t = base[0, sl]
    t_in = hm.second_preimage(t, ens_seed(band, 0), rs)             # same fingerprint in partition 0, other tuple
    t_x = hm.tuple_with_state(hm._state([int(v) for v in t], ens_seed(band, 0)), ens_seed(band, 1), r, rs)
    e0 = hm.tuple_with_prefp(hm.EMPTY_KEY, ens_seed(0, 0), r, rs)   # the empty-key tuple in band 0 of partition 0
    assert t_in is not None and t_x is not None and e0 is not None
    assert ens_fp(t_in[None], band, 0)[0] == ens_fp(t[None], band, 0)[0] == ens_fp(t_x[None], band, 1)[0]
    assert ens_fp(t[None], band, 1)[0] != ens_fp(t[None], band, 0)[0]
    rows, sizes = [base[0]], [s0]
    for tt, size in ((t, s0), (t, s1), (t_in, s0), (t_in, s0), (t_x, s1), (t_x, s1)):
        x = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
        x[sl] = tt
        rows.append(x)
        sizes.append(size)
    for _ in range(2):
        x = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
        x[0:r] = e0
        rows.append(x)
        sizes.append(s0)
    extra = [base[j] for j in range(1, 20)]
    if head_collides:
        rows, sizes = extra + rows, [s0 if j % 2 else s1 for j in range(19)] + sizes
    else:
        rows, sizes = rows + extra, sizes + [s0 if j % 2 else s1 for j in range(19)]
    rows = np.stack(rows)
    qs = []
    for tt in (t, t_in, t_x, e0):
        x = rs.randint(0, 1 << 32, size=k, dtype=np.uint64).astype(np.uint32)
        if tt is e0:
            x[0:r] = tt
        else:
            x[sl] = tt
        qs.append(x)
    qsig = np.stack(qs)
    qsize = _sizes_for(host, s0, row)
    assert np.searchsorted(host.xqs, s1 / qsize) == row
    try:
        _, want = _check(ens, rows, sizes, qsig, [qsize] * 4)
        off = 19 if head_collides else 0
        assert set(want[0]) == {off + 0, off + 1, off + 2}          # t: its own rows in both partitions, nothing else
        assert set(want[1]) == {off + 3, off + 4}
        assert set(want[2]) == {off + 5, off + 6}
        assert set(want[3]) == {off + 7, off + 8}
    finally:
        ens.close()


def test_one_set_no_queries_extreme_sizes(be):
    k = 32
    ens = be.ensemble(0.5, k, 4, 4)
    row = np.arange(k, dtype=np.uint32)[None]
    try:
        ptr, idx, eq = ens.query(row, [5])                          # nothing indexed yet
        assert ptr.tolist() == [0, 0] and len(idx) == 0
        _check(ens, row, [7], np.concatenate([row, row, row]), [1, 7, 10 ** 12])
        got = _got(*ens.query(np.concatenate([row, row, row]), [1, 7, 10 ** 12]))
        assert got == [{0: k}, {0: k}, {0: k}]
        ptr, idx, eq = ens.query(np.zeros((0, k), dtype=np.uint32), np.zeros(0, dtype=np.int64))
        assert ptr.tolist() == [0] and len(idx) == 0 and len(eq) == 0
    finally:
        ens.close()


def test_more_items_than_one_grid_sweep(be):
    """(query, partition) items beyond one sweep of the grid."""
    k = 32
    rs = np.random.RandomState(9)
    n = 200 if be.name == "emu" else 4000
    sig = _low_entropy(rs, n, k, 3)
    sizes = rs.randint(1, 400, n)
    nq = (3 * be.grid_items) // 8 + 5
    qsig = sig[rs.randint(0, n, nq)]
    ens = be.ensemble(0.4, k, 8, 4)
    try:
        _check(ens, sig, sizes, qsig, rs.randint(1, 400, nq))
    finally:
        ens.close()


def test_c_abi_argument_validation(emu_lib):
    lib, k = emu_lib, 32
    buf = _aligned(np.zeros(256, dtype=np.int64))
    b = np.array([4, 8], dtype=np.int32)
    r = np.array([2, 4], dtype=np.int32)
    h = ctypes.c_void_p()
    for args in ((1, 4, _p(b), _p(r), 2), (k, 0, _p(b), _p(r), 2), (k, 4, _p(b), _p(r), 0), (k, 4, _p(b), _p(r), 17),
                 (k, 4, None, _p(r), 2), (k, 4, _p(b), None, 2)):
        assert lib.dsk_lsh_ensemble_create(*args, 0, ctypes.byref(h)) == DSK_ERR_INVALID
    for bad in (np.array([0, 8], dtype=np.int32), np.array([17, 8], dtype=np.int32)):   # b < 1, b * r > K
        assert lib.dsk_lsh_ensemble_create(k, 4, _p(bad), _p(r), 2, 0, ctypes.byref(h)) == DSK_ERR_INVALID
        assert b"(b, r) table" in lib.dsk_last_error()
    assert lib.dsk_lsh_ensemble_create(k, 2, _p(b), _p(r), 2, 0, None) == DSK_ERR_INVALID
    assert lib.dsk_lsh_ensemble_size(None, None) == DSK_ERR_INVALID
    assert lib.dsk_lsh_ensemble_index_bytes(None, 10) == 0
    assert lib.dsk_lsh_ensemble_create(k, 2, _p(b), _p(r), 2, 0, ctypes.byref(h)) == DSK_OK
    try:
        n = 10
        cap = 32                                                     # the power of two >= 2n
        assert lib.dsk_lsh_ensemble_index_bytes(h, n) == 4 * k * n + 4 * n + 8 * 3 + (k // 2) * (16 * cap + 4 * n) + \
            (k // 4) * (16 * cap + 4 * n)
        sig = _aligned(np.arange(n * k, dtype=np.uint32).reshape(n, k) % 3)
        order = _aligned(np.arange(n, dtype=np.int32))
        for start in ([0, 5, 9], [1, 5, 10], [0, 6, 5, 10][:3], [0, 11, 10]):
            st = np.array(start, dtype=np.int64)
            assert lib.dsk_lsh_ensemble_index(h, _p(sig), n, _p(order), _p(st), None) == DSK_ERR_INVALID
            assert b"h_part_start" in lib.dsk_last_error()
        st = np.array([0, 5, 10], dtype=np.int64)
        for args in ((None, _p(sig), n, _p(order), _p(st)), (h, None, n, _p(order), _p(st)), (h, _p(sig), n, None, _p(st)),
                     (h, _p(sig), n, _p(order), None), (h, _p(sig), 0, _p(order), _p(st)),
                     (h, _p(sig), 1 << 31, _p(order), _p(st))):
            assert lib.dsk_lsh_ensemble_index(*args, None) == DSK_ERR_INVALID
        sz = ctypes.c_int64(-1)
        assert lib.dsk_lsh_ensemble_size(h, ctypes.byref(sz)) == DSK_OK and sz.value == 0
        assert lib.dsk_lsh_ensemble_index(h, _p(sig), n, _p(order), _p(st), None) == DSK_OK
        assert lib.dsk_lsh_ensemble_size(h, ctypes.byref(sz)) == DSK_OK and sz.value == n
        assert lib.dsk_lsh_ensemble_index(h, _p(sig), n, _p(order), _p(st), None) == DSK_ERR_INVALID
        assert b"Cannot call index again" in lib.dsk_last_error()
        for fn, nb in ((lib.dsk_lsh_ensemble_query_count, 1), (lib.dsk_lsh_ensemble_query_fill, 2)):
            tail = [None] if fn is lib.dsk_lsh_ensemble_query_fill else []
            assert fn(None, _p(buf), 1, _p(buf), *[_p(buf)] * nb, *tail, None) == DSK_ERR_INVALID
            assert b"null handle" in lib.dsk_last_error()
            assert fn(h, _p(buf), -1, _p(buf), *[_p(buf)] * nb, *tail, None) == DSK_ERR_INVALID
            assert b"nq must be" in lib.dsk_last_error()
            assert fn(h, None, 1, _p(buf), *[_p(buf)] * nb, *tail, None) == DSK_ERR_INVALID
            assert fn(h, _p(buf), 1, None, *[_p(buf)] * nb, *tail, None) == DSK_ERR_INVALID
            for j in range(nb):
                args = [_p(buf)] * nb
                args[j] = None
                assert fn(h, _p(buf), 1, _p(buf), *args, *tail, None) == DSK_ERR_INVALID
                assert b"null buffer" in lib.dsk_last_error()
            assert fn(h, None, 0, None, *[None] * nb, *tail, None) == DSK_OK
        # selection values outside the table skip the partition
        q = _aligned(np.asarray(sig[:1]))
        sel = _aligned(np.array([-1, 2], dtype=np.int32))
        cnt = _aligned(np.full(2, -7, dtype=np.int64))
        assert lib.dsk_lsh_ensemble_query_count(h, _p(q), 1, _p(sel), _p(cnt), None) == DSK_OK and cnt.tolist() == [0, 0]
        sel = _aligned(np.array([1, 0], dtype=np.int32))
        assert lib.dsk_lsh_ensemble_query_count(h, _p(q), 1, _p(sel), _p(cnt), None) == DSK_OK and cnt[0] >= 1
    finally:
        lib.dsk_lsh_ensemble_destroy(h)
    lib.dsk_lsh_ensemble_destroy(None)


def test_constructor_errors_and_params():
    """The constructor checks and the (b, r) table are the host class's (no device needed: they run first)."""
    import datasketch_b200 as dsk
    for kw in [dict(threshold=1.5), dict(threshold=-0.1), dict(num_perm=1), dict(num_part=0), dict(m=1),
               dict(m=200, num_perm=128), dict(weights=(1.5, -0.5)), dict(weights=(0.3, 0.3))]:
        with pytest.raises(ValueError) as e_gpu:
            dsk.GpuLSHEnsemble(**kw)
        with pytest.raises(ValueError) as e_host:
            dsk.MinHashLSHEnsemble(**kw)
        assert str(e_gpu.value) == str(e_host.value)


# ---- GPU only ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_api_keys_errors_and_outputs():
    import torch
    import datasketch_b200 as dsk
    rs = np.random.RandomState(4)
    k = 64
    sig = _low_entropy(rs, 300, k, 3)
    sizes = rs.randint(1, 100, 300)
    ens = dsk.GpuLSHEnsemble(threshold=0.5, num_perm=k, num_part=8, m=4)
    host = dsk.MinHashLSHEnsemble(threshold=0.5, num_perm=k, num_part=8, m=4)
    assert np.array_equal(ens.params, host.params) and np.array_equal(ens.xqs, host.xqs)
    assert ens.is_empty() and len(ens) == 0 and 0 not in ens
    with pytest.raises(ValueError, match="entries is empty"):
        ens.index(np.zeros((0, k), dtype=np.uint32), [])
    with pytest.raises(ValueError, match="Set size must be positive"):
        ens.index(sig, np.where(np.arange(300) == 7, 0, sizes))
    with pytest.raises(ValueError, match="Expecting minhash with length"):
        ens.index(sig[:, :k - 1], sizes)
    with pytest.raises(ValueError):
        ens.index(sig, sizes[:-1])
    with pytest.raises(ValueError):
        ens.index(sig, sizes, keys=["x"] * 5)
    assert ens.is_empty()
    keys = ["k%d" % i for i in range(300)]
    ens.index(torch.from_numpy(sig.view(np.int32)).cuda(), torch.from_numpy(sizes), keys=keys)
    assert len(ens) == 300 and not ens.is_empty() and "k0" in ens and "k299" in ens and "k300" not in ens
    with pytest.raises(ValueError, match="Cannot call index again"):
        ens.index(sig, sizes)
    q = sig[:50]
    qs = rs.randint(1, 100, 50)
    with pytest.raises(ValueError, match="Set size must be positive"):
        ens.query(q, np.zeros(50, dtype=np.int64))
    with pytest.raises(ValueError, match="Expecting minhash with length"):
        ens.query(np.zeros((2, k + 1), dtype=np.uint32), [1, 1])
    with pytest.raises(TypeError):
        ens.query(torch.zeros((2, k), dtype=torch.int64, device="cuda"), [1, 1])
    ptr, idx = ens.query(q, qs)
    orc = Oracle(host, sig, sizes.tolist())
    assert [set(g) for g in _got(ptr, idx)] == [set(w) for w in _want(orc, sig, q, qs)]
    assert [sorted(x) for x in ens.query_keys(q, qs)] == [sorted(keys[i] for i in w) for w in _want(orc, sig, q, qs)]
    p2, i2, e2 = ens.query(torch.from_numpy(q.view(np.int32)).cuda(), qs, with_eq=True, to_host=False)
    assert p2.is_cuda and p2.dtype == torch.int64 and i2.dtype == torch.int32 and e2.dtype == torch.int32
    assert np.array_equal(p2.cpu().numpy(), ptr)
    ens2 = dsk.GpuLSHEnsemble(threshold=0.5, num_perm=k, num_part=8, m=4)
    ens2.index(sig, sizes)
    assert 0 in ens2 and 299 in ens2 and 300 not in ens2
    assert [sorted(x) for x in ens2.query_keys(q, qs)] == [sorted(w) for w in _want(orc, sig, q, qs)]   # row numbers


@pytest.mark.gpu
def test_scale_one_million_sets_10k_queries():
    """1M sets (K = 128, heavy-tailed sizes, the default-like configuration 0.5 / 16 partitions / m = 8) and 10k
    queries; a sample of queries is checked against a brute-force torch computation of the definition: band-tuple
    equality over each partition's rows, independent of the hash tables."""
    import torch
    import datasketch_b200 as dsk
    n, k, nq = 1_000_000, 128, 10_000
    g = torch.Generator(device="cuda").manual_seed(3)
    sig = torch.randint(0, 64, (n, k), dtype=torch.int32, device="cuda", generator=g)   # low entropy: real buckets
    sig[:, 16:] = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, k - 16), dtype=torch.int32, device="cuda", generator=g)
    rs = np.random.RandomState(3)
    sizes = np.clip((rs.pareto(1.2, n) * 50 + 10).astype(np.int64), 10, 100_000)
    mag = 10 ** np.maximum(np.floor(np.log10(sizes)).astype(np.int64) - 1, 0)
    sizes = sizes // mag * mag             # two significant digits: the host partitioner is quadratic in distinct sizes
    src = torch.randint(0, n, (nq,), device="cuda", generator=g)
    qsig = sig[src].clone()
    qsig[nq // 2:, 16:] = torch.randint(-2 ** 31, 2 ** 31 - 1, (nq - nq // 2, k - 16), dtype=torch.int32, device="cuda",
                                        generator=g)
    qsizes = np.clip((rs.pareto(1.2, nq) * 50 + 1).astype(np.int64), 1, 10 ** 6)
    ens = dsk.GpuLSHEnsemble(threshold=0.5, num_perm=k, num_part=16, m=8)
    ens.index(sig, sizes)
    ptr, idx, eq = ens.query(qsig, qsizes, with_eq=True)
    assert ptr[-1] >= nq
    part = np.repeat(np.arange(16), np.diff(ens._start))
    part_of = np.empty(n, dtype=np.int64)
    part_of[np.argsort(sizes, kind="stable")] = part
    part_of = torch.from_numpy(part_of).cuda()
    sel = ens.selection(qsizes)
    for q in np.random.RandomState(1).choice(nq, 64, replace=False).tolist():
        hit = torch.zeros(n, dtype=torch.bool, device="cuda")
        for p in range(16):
            if sel[q, p] < 0:
                continue
            b, r = (int(x) for x in ens.params[sel[q, p]])
            rows = (part_of == p)
            eqpos = (sig[:, :b * r] == qsig[q, :b * r]).view(n, b, r).all(dim=2).any(dim=1)
            hit |= rows & eqpos
        want = set(torch.nonzero(hit).flatten().tolist())
        got = idx[ptr[q]:ptr[q + 1]].tolist()
        assert len(got) == len(want) and set(got) == want, q
        want_eq = (sig[got] == qsig[q]).sum(dim=1).cpu().numpy() if got else np.zeros(0)
        assert np.array_equal(eq[ptr[q]:ptr[q + 1]], want_eq)
