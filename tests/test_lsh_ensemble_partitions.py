"""The size partitioner of MinHashLSHEnsemble on the device (``dsk_ensemble_partition``, ``optimal_partitions_device``).

Its bounds must be the reference's ``optimal_partitions`` (lshensemble_partition.py) for every input, so every cost must be
the reference's float64 value bit for bit: each term rounded operation by operation, each sum numpy's pairwise sum; the
dynamic programme and the back-tracking as the reference runs them (the back-tracking reads the p-interval table where the
recurrence used p-1, and its zero entries); every argmin the first index among equal values.

tests/golden/ensemble_partitions.npz (oracle/gen_golden_ensemble_partitions.py) holds the reference's own cost triangles
(SHA-256 digests of their bit patterns, and the bits themselves up to D = 64) and bounds, over heavy-tailed and tie-rich
distributions and a sweep where the back-tracking quirk changes the bounds.  The CPU tests run the whole library on the
emulation shim through its C-ABI; the ``gpu`` tests run the same checks, larger sweeps against the host
``optimal_partitions`` and D = 20000 / 30000 on the H100.
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_lsh_self_join import _aligned, _p  # noqa: E402

from datasketch_b200 import lshensemble as le  # noqa: E402

SIZE_MAX = 2 ** 64 - 1


def _triangle(cost):
    """The column-major upper triangle of a full D x D matrix: entry (l, u) at u(u+1)/2 + l."""
    n = cost.shape[0]
    return np.concatenate([cost[:u + 1, u] for u in range(n)])


def _fixture(golden):
    """``dists[d] = (sizes, counts, ref)`` with ref = (SHA-256 of the reference's triangle, the triangle's bits or None) and
    ``cases[c] = (d, num_part, quirk, lowers, uppers)``."""
    g = golden("ensemble_partitions")
    dp, cp = g["dist_ptr"], g["case_ptr"]
    dists = [(g["sizes"][dp[i]:dp[i + 1]], g["counts"][dp[i]:dp[i + 1]],
              (str(g["cost_sha256"][i]), g["d%d_cost" % i] if "d%d_cost" % i in g else None)) for i in range(len(dp) - 1)]
    cases = [(int(d), int(k), bool(q), g["lowers"][cp[c]:cp[c + 1]], g["uppers"][cp[c]:cp[c + 1]])
             for c, (d, k, q) in enumerate(g["cases"])]
    return dists, cases


def _is_reference_triangle(tri, ref):
    """``tri`` (float64, column-major upper triangle) is the reference's, bit for bit: its digest, and its bits where the
    fixture holds them."""
    bits = np.ascontiguousarray(tri).view(np.uint64)
    digest, want = ref
    return hashlib.sha256(bits.astype("<u8").tobytes()).hexdigest() == digest and (want is None or np.array_equal(bits, want))


def _emu_partition(lib, sizes, counts, num_part, with_cost=False):
    """``(upper indices, cost triangle or None)`` from the emulated C-ABI."""
    sizes = _aligned(np.asarray(sizes, dtype=np.int64))
    counts = _aligned(np.asarray(counts, dtype=np.int64))
    n = len(sizes)
    need = int(lib.dsk_ensemble_partition_workspace_size(n, num_part))
    ws = _aligned(np.zeros(max(need, 16), dtype=np.uint8))
    cost = _aligned(np.full(n * (n + 1) // 2, np.nan)) if with_cost else None
    upper = np.full(max(min(num_part, n), 1), -7, dtype=np.int64)
    rc = lib.dsk_ensemble_partition(_p(sizes), _p(counts), n, num_part, _p(ws), need, 0, _p(upper),
                                    _p(cost) if with_cost else None, None)
    assert rc == 0, lib.dsk_last_error()
    return upper, cost


def _bounds(sizes, upper):
    lowers = np.concatenate([[0], upper[:-1] + 1])
    return [(int(sizes[a]), int(sizes[b])) for a, b in zip(lowers, upper)]


def _host_bounds(sizes, counts, num_part):
    return [(int(a), int(b)) for a, b in le.optimal_partitions(sizes, counts, num_part)]


def _random_dist(rs, d, top=10 ** 9):
    sizes = np.unique(rs.randint(1, top, 2 * d + 16).astype(np.int64))
    sizes = np.sort(rs.choice(sizes, d, replace=False))
    counts = np.minimum((rs.pareto(0.9, d) * 4 + 1).astype(np.int64), 10 ** 7)
    return sizes, counts


# ---- the emulated library (CPU) ----------------------------------------------------------------------------------------
def test_fixture_covers_what_it_claims(golden):
    dists, cases = _fixture(golden)
    ds = {len(s) for s, _, _ in dists}
    assert {1, 2, 7, 8, 9, 64, 128, 129, 136, 257, 400} <= ds
    assert sum(int(s.max()) == 10 ** 9 for s, _, _ in dists) >= 9      # sizes up to 10^9
    for d_want in (64, 400):
        i = [j for j, (s, _, _) in enumerate(dists) if len(s) == d_want][0]
        assert {k for d, k, _, _, _ in cases if d == i} == {1, 2, 3, 8, 16, 32, d_want - 1, d_want, d_want + 1}
    assert sum(q for _, _, q, _, _ in cases) >= 50      # the back-tracking quirk changes these bounds


def test_host_partitioner_is_the_reference(golden):
    """The host restatement (the tests' reference below) gives the fixture's triangles and bounds."""
    dists, cases = _fixture(golden)
    for sizes, counts, ref in dists:
        if len(sizes) <= 136:
            assert _is_reference_triangle(_triangle(le._interval_costs(sizes, counts)), ref), len(sizes)
    for d, k, _, lo, up in cases:
        if len(dists[d][0]) <= 64:
            assert _host_bounds(dists[d][0], dists[d][1], k) == list(zip(lo.tolist(), up.tolist()))


def test_emu_cost_triangle_bit_equal(emu_lib, golden):
    """The device triangle equals the reference's _compute_nfps_real bit for bit, and the host _interval_costs."""
    dists, _ = _fixture(golden)
    for sizes, counts, ref in dists:
        _, cost = _emu_partition(emu_lib, sizes, counts, 1, with_cost=True)
        assert _is_reference_triangle(cost, ref), len(sizes)
        if len(sizes) in (129, 257):
            assert np.array_equal(cost.view(np.uint64), _triangle(le._interval_costs(sizes, counts)).view(np.uint64))


def test_emu_bounds_equal_fixture(emu_lib, golden):
    """The cases of the fixture: heavy-tailed, tie-rich, num_part from 1 to D + 1, the quirk sweep.  The triangle written
    with the bounds is the fixture's too.  The emulation runs one host thread per CUDA thread and each of the num_part - 2
    programme steps is a launch, so num_part near D is run here up to D = 64 (the H100 test runs every case)."""
    dists, cases = _fixture(golden)
    for d, k, _, lo, up in cases:
        sizes, counts, ref = dists[d]
        if k > 32 and k < len(sizes) and len(sizes) > 64:
            continue
        upper, cost = _emu_partition(emu_lib, sizes, counts, k, with_cost=len(sizes) == 64)
        assert _bounds(sizes, upper) == list(zip(lo.tolist(), up.tolist())), (len(sizes), k)
        if cost is not None:
            assert _is_reference_triangle(cost, ref)


@pytest.mark.parametrize("seed", range(6))
def test_emu_random_sweep_against_host_partitioner(emu_lib, seed):
    """Seeded distributions (heavy-tailed counts; also small sizes and counts, where equal totals are common) against the
    host optimal_partitions, bounds and triangle."""
    rs = np.random.RandomState(100 + seed)
    d = int(rs.randint(3, 140))
    sizes, counts = _random_dist(rs, d) if seed % 2 else (np.sort(rs.choice(np.arange(1, 200), d, replace=False)),
                                                           rs.randint(1, 4, d).astype(np.int64))
    host_cost = le._interval_costs(sizes, counts)
    for k in sorted({2, 3, int(rs.randint(2, min(d, 24))), min(16, d - 1), d - 1 if d < 40 else 2}):
        if k < 2:
            continue
        upper, cost = _emu_partition(emu_lib, sizes, counts, k, with_cost=True)
        assert _bounds(sizes, upper) == _host_bounds(sizes, counts, k), (d, k)
        assert np.array_equal(cost.view(np.uint64), _triangle(host_cost).view(np.uint64))


def test_emu_index_plan_with_device_partitioner(emu_lib):
    """_index_plan over a partitioner with optimal_partitions' contract: the emulated device one gives the host plan."""
    def emu_partitioner(vals, counts, k):
        upper, _ = _emu_partition(emu_lib, vals, counts, k)
        if k < 2:
            return [(vals[0], vals[-1])]
        if k >= len(vals):
            return [(x, x) for x in vals]
        return [(vals[a], vals[b]) for a, b in zip(np.concatenate([[0], upper[:-1] + 1]), upper)]

    rs = np.random.RandomState(5)
    for n, top, k in ((300, 90, 16), (500, 400, 8), (50, 5, 16), (40, 200, 1), (2000, 120, 32)):
        sizes = (rs.pareto(1.2, n) * 3 + 1).astype(np.int64) % top + 1
        want = le._index_plan(sizes, k)
        got = le._index_plan(sizes, k, emu_partitioner)
        assert want[0] == got[0] and want[1] == got[1]
        assert np.array_equal(want[2], got[2]) and np.array_equal(want[3], got[3])


def test_emu_c_abi_validation_and_workspace_size(emu_lib):
    lib = emu_lib
    ws_size = lib.dsk_ensemble_partition_workspace_size
    assert ws_size(0, 4) == 0 and ws_size(5, 0) == 0 and ws_size(-1, 4) == 0
    r = lambda x: (x + 255) // 256 * 256  # noqa: E731
    assert ws_size(10, 1) == r(160) and ws_size(10, 10) == r(160)              # no table: sizes and counts only
    assert ws_size(10, 4) == r(160) + r(8 * 55) + r(8 * 10 * 3) + r(32)
    big = 30000                                                                  # the terms leave shared memory
    assert ws_size(big, 16) == r(16 * big) + r(8 * big * 512) + r(4 * big * (big + 1)) + r(8 * big * 15) + r(128)
    assert ws_size(3550, 16) == r(16 * 3550) + r(4 * 3550 * 3551) + r(8 * 3550 * 15) + r(128)
    assert ws_size(1 << 32, 16) == SIZE_MAX and ws_size(1 << 62, 2) == SIZE_MAX and ws_size(2 ** 63 - 1, 16) == SIZE_MAX
    assert ws_size(1 << 62, 1) == SIZE_MAX                                       # 16 * D alone overflows

    def call(sizes, counts, k, ws_bytes=None, misalign=0, n=None):
        sizes = _aligned(np.asarray(sizes, dtype=np.int64))
        counts = _aligned(np.asarray(counts, dtype=np.int64))
        n = len(sizes) if n is None else n
        need = int(ws_size(max(n, 1), max(k, 1)))
        ws = _aligned(np.zeros(need + 64, dtype=np.uint8))
        out = np.zeros(max(len(sizes), k, 1), dtype=np.int64)
        rc = lib.dsk_ensemble_partition(_p(sizes), _p(counts), n, k, ws.ctypes.data + misalign,
                                        need if ws_bytes is None else ws_bytes, 0, _p(out), None, None)
        return rc, lib.dsk_last_error().decode(), out

    s, c = [1, 5, 9, 12, 40], [3, 1, 4, 1, 5]
    assert call(s, c, 3)[0] == 0
    for args, msg in (((s, c, 0), "num_part >= 1"), ((s, c, 3, None, 0, 0), "n_sizes >= 1"),
                      (([1, 5, 5, 12, 40], c, 3), "strictly ascending"), (([1, 9, 5, 12, 40], c, 3), "strictly ascending"),
                      (([0, 5, 9, 12, 40], c, 3), "strictly ascending"), (([-3, 5, 9, 12, 40], c, 3), "[1, 2^62)"),
                      (([1, 5, 9, 12, 1 << 62], c, 3), "[1, 2^62)"), ((s, [3, 1, 0, 1, 5], 3), "counts"),
                      ((s, [3, 1, -2, 1, 5], 3), "counts"), ((s, [3, 1, 1 << 62, 1, 5], 3), "counts"),
                      ((s, c, 3, 100), "workspace"), ((s, c, 3, None, 8), "16-byte aligned")):
        rc, err, _ = call(*args)
        assert rc == 1 and msg in err, (args, err)
    assert call(s, c, 3, None, 16)[0] == 0                                   # any 16-byte alignment will do
    assert call([1, 5, 9, 12, (1 << 62) - 1], [1, 1, 1, 1, (1 << 62) - 1], 3)[0] == 0
    # no table: the trivial bounds on the host, no workspace needed
    out = np.zeros(5, dtype=np.int64)
    a, b = _aligned(np.array(s, dtype=np.int64)), _aligned(np.array(c, dtype=np.int64))
    assert lib.dsk_ensemble_partition(_p(a), _p(b), 5, 1, None, 0, 0, _p(out), None, None) == 0 and out[0] == 4
    assert lib.dsk_ensemble_partition(_p(a), _p(b), 5, 9, None, 0, 0, _p(out), None, None) == 0
    assert out.tolist() == [0, 1, 2, 3, 4]
    assert lib.dsk_ensemble_partition(_p(a), _p(b), 5, 3, None, 0, 0, _p(out), None, None) == 1
    assert lib.dsk_ensemble_partition(None, _p(b), 5, 3, None, 0, 0, _p(out), None, None) == 1
    assert "null buffer" in lib.dsk_last_error().decode()


# ---- the H100 ------------------------------------------------------------------------------------------------------------
def _dev_partition(sizes, counts, num_part, with_cost):
    """The C-ABI on cuda:0 with torch buffers: (upper indices, triangle as float64 numpy or None)."""
    import torch
    from datasketch_b200 import _native as nv
    lib = nv.load()
    s = np.ascontiguousarray(sizes, dtype=np.int64)
    c = np.ascontiguousarray(counts, dtype=np.int64)
    n = len(s)
    need = int(lib.dsk_ensemble_partition_workspace_size(n, num_part))
    ws = torch.empty((max(need, 16),), dtype=torch.uint8, device="cuda:0")
    cost = torch.full((n * (n + 1) // 2,), float("nan"), dtype=torch.float64, device="cuda:0") if with_cost else None
    out = np.zeros(max(min(num_part, n), 1), dtype=np.int64)
    nv.check(lib.dsk_ensemble_partition(s.ctypes.data, c.ctypes.data, n, num_part, ws.data_ptr(), need, 0, out.ctypes.data,
                                        cost.data_ptr() if with_cost else None, torch.cuda.current_stream().cuda_stream))
    return out, cost


@pytest.mark.gpu
def test_gpu_fixture(golden):
    dists, cases = _fixture(golden)
    for sizes, counts, ref in dists:
        _, cost = _dev_partition(sizes, counts, 1, True)
        assert _is_reference_triangle(cost.cpu().numpy(), ref), len(sizes)
    for d, k, _, lo, up in cases:
        sizes, counts, _ = dists[d]
        got = le.optimal_partitions_device(sizes, counts, k)
        assert [(int(a), int(b)) for a, b in got] == list(zip(lo.tolist(), up.tolist())), (len(sizes), k)
        if len(sizes) <= 64:   # the same list, element types included
            assert got == le.optimal_partitions(sizes, counts, k)


@pytest.mark.gpu
@pytest.mark.parametrize("d,seed", [(1000, 0), (1499, 1)])
def test_gpu_random_sweep_against_host(d, seed, monkeypatch):
    """D = 1000 / 1499 against the host optimal_partitions (its cost table computed once per distribution), bounds and full
    triangle."""
    rs = np.random.RandomState(seed)
    sizes, counts = _random_dist(rs, d)
    host_cost = le._interval_costs(sizes, counts)
    monkeypatch.setattr(le, "_interval_costs", lambda s, c: host_cost)
    _, cost = _dev_partition(sizes, counts, 16, True)
    assert np.array_equal(cost.cpu().numpy().view(np.uint64), _triangle(host_cost).view(np.uint64))
    for k in (2, 3, 16, 32, int(rs.randint(4, 200))):
        assert le.optimal_partitions_device(sizes, counts, k) == le.optimal_partitions(sizes, counts, k), k


@pytest.mark.gpu
@pytest.mark.parametrize("d", [20000, 30000])
def test_gpu_large_d_sampled_columns(d):
    """D = 20000 (a column's terms in shared memory) and 30000 (in global memory): sampled columns, the first and last
    included, equal numpy's per-entry np.sum bit for bit; the bounds are ascending, cover the domain and number num_part."""
    import torch
    rs = np.random.RandomState(d)
    sizes, counts = _random_dist(rs, d)
    upper, cost = _dev_partition(sizes, counts, 16, True)
    cols = [0, 1, 7, 8, 127, 128, 129, 1000, 8193, d // 2, d - 2, d - 1] if d == 20000 else [0, 129, 28671, 28672, d - 1]
    for u in cols:
        start = u * (u + 1) // 2
        got = cost[start:start + u + 1].cpu().numpy()
        top = float(sizes[u])
        want = np.array([np.sum((top - sizes[l:u + 1]) / top * counts[l:u + 1]) for l in range(u + 1)])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), u
    del cost
    torch.cuda.empty_cache()
    assert len(upper) == 16 and upper[-1] == d - 1 and upper[0] >= 0 and np.all(np.diff(upper) > 0)
    got = le.optimal_partitions_device(sizes, counts, 16)
    assert got == _bounds(sizes, upper) and got[0][0] == sizes[0] and got[-1][1] == sizes[-1]


@pytest.mark.gpu
def test_gpu_index_uses_the_device_partitioner():
    """GpuLSHEnsemble.index on seeded corpora: lowers / uppers / _start are those of the host plan."""
    from datasketch_b200.lshensemble import GpuLSHEnsemble, _index_plan
    rs = np.random.RandomState(11)
    for n, top, num_part in ((5000, 3000, 16), (800, 40, 8), (300, 7, 16), (1000, 500, 1), (20000, 600, 32)):
        sizes = (rs.pareto(1.1, n) * 5 + 1).astype(np.int64) % top + 1
        sig = rs.randint(0, 2 ** 32, size=(n, 32), dtype=np.uint64).astype(np.uint32)
        ens = GpuLSHEnsemble(threshold=0.5, num_perm=32, num_part=num_part, m=4)
        ens.index(sig, sizes)
        lowers, uppers, _, start = _index_plan(sizes, num_part)
        assert ens.lowers == lowers and ens.uppers == uppers and np.array_equal(ens._start, start), (n, top)


@pytest.mark.gpu
def test_gpu_errors():
    from datasketch_b200.lshensemble import GpuLSHEnsemble
    s, c = np.array([1, 5, 9, 12, 40]), np.array([3, 1, 4, 1, 5])
    assert le.optimal_partitions_device(s, c, 3) == le.optimal_partitions(s, c, 3)
    assert le.optimal_partitions_device(s, c, 1) == le.optimal_partitions(s, c, 1)
    assert le.optimal_partitions_device(s, c, 7) == le.optimal_partitions(s, c, 7)
    assert le.optimal_partitions_device(list(s), list(c), 2) == le.optimal_partitions(s, c, 2)
    with pytest.raises(ValueError, match="strictly ascending"):
        le.optimal_partitions_device([1, 9, 5, 12, 40], c, 3)
    with pytest.raises(ValueError, match="strictly ascending"):
        le.optimal_partitions_device([1, 9, 9, 12, 40], c, 1)
    with pytest.raises(ValueError, match="counts"):
        le.optimal_partitions_device(s, [3, 1, 0, 1, 5], 3)
    with pytest.raises(ValueError):
        le.optimal_partitions_device(s, c, 0)
    with pytest.raises(ValueError):
        le.optimal_partitions_device(s, c[:4], 3)
    with pytest.raises(ValueError):
        le.optimal_partitions_device([], [], 3)
    with pytest.raises(TypeError):
        le.optimal_partitions_device(s.astype(float), c, 3)
    big = np.arange(1, 200001, dtype=np.int64)
    with pytest.raises(MemoryError, match="D = 200000"):
        le.optimal_partitions_device(big, np.ones_like(big), 16)
    # index: MemoryError, the object stays empty and indexes afterwards
    ens = GpuLSHEnsemble(threshold=0.5, num_perm=16, num_part=16, m=4)
    sig = np.random.RandomState(0).randint(0, 2 ** 32, size=(len(big), 16), dtype=np.uint64).astype(np.uint32)
    with pytest.raises(MemoryError):
        ens.index(sig, big)
    assert ens.is_empty() and ens.uppers == [None] * 16
    ens.index(sig[:1000], big[:1000] % 97 + 1)
    assert len(ens) == 1000 and ens.uppers[-1] == 97
