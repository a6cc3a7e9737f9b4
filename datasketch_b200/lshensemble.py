"""MinHashLSHEnsemble (containment search) with the reference's API (datasketch/lshensemble.py:61-265,
datasketch/lshensemble_partition.py), on top of this package's ``MinHashLSH``.

What runs where:

* parameter tables (``_optimal_param``: scipy ``quad`` over ten x/q ratios) are host-side control logic, float64, the
  same expressions in the same order as the reference so the chosen (b, r) are identical;
* the size partitioner (dynamic programme over the distinct set sizes) has two implementations with the reference's
  bounds: ``optimal_partitions`` on the host (``MinHashLSHEnsemble``, and the tests' reference) and
  ``optimal_partitions_device``, whose cost table (cubic in the number of distinct sizes), dynamic programme and
  back-tracking run on the device (``dsk_ensemble_partition``; ``GpuLSHEnsemble.index`` uses it);
* ``index`` inserts each partition's sets into its ``MinHashLSH`` instances with ``insert_batch``: the band keys of
  the whole partition come from one ``dsk_band_keys`` launch per distinct r instead of one ``_H`` call per set
  and band (lshensemble.py:221-228 -> lsh.py:344);
* ``query`` probes the first b bands of each partition's index (``MinHashLSH._query_b``), as the reference does.
"""
from __future__ import annotations

import ctypes
import random
import string
import struct
from collections import Counter
from typing import Dict, Generator, Hashable, Iterable, List, Optional, Tuple

import numpy as np
from scipy.integrate import quad as integrate

from .lsh import MinHashLSH
from .minhash import MinHash


def _random_name(length: int) -> bytes:
    """Default storage basename: random lowercase letters, as bytes (storage.py:1052-1054)."""
    return "".join(random.choice(string.ascii_lowercase) for _ in range(length)).encode("utf8")


# ---- (b, r) for a containment threshold and a size ratio xq = x / q (lshensemble.py:17-58) -------------------
def _false_positive_probability(threshold: float, b: int, r: int, xq: float) -> float:
    """Area under the collision-probability curve below the threshold; containment t maps to the Jaccard
    similarity t / (1 + xq - t), and t cannot exceed xq."""
    prob = lambda t: 1 - (1 - (t / (1 + xq - t)) ** float(r)) ** float(b)  # noqa: E731
    area, _ = integrate(prob, 0.0, threshold if xq >= threshold else xq)
    return area


def _false_negative_probability(threshold: float, b: int, r: int, xq: float) -> float:
    prob = lambda t: 1 - (1 - (1 - (t / (1 + xq - t)) ** float(r)) ** float(b))  # noqa: E731
    if xq >= 1.0:
        return integrate(prob, threshold, 1.0)[0]
    if xq >= threshold:
        return integrate(prob, threshold, xq)[0]
    return 0.0


def _optimal_param(threshold: float, num_perm: int, max_r: int, xq: float, false_positive_weight: float,
                   false_negative_weight: float) -> Tuple[int, int]:
    """Grid search over b in [1, num_perm], r in [1, max_r], b*r <= num_perm; first strict minimum wins."""
    best, opt = float("inf"), (0, 0)
    for b in range(1, num_perm + 1):
        for r in range(1, max_r + 1):
            if b * r > num_perm:
                continue
            err = (_false_positive_probability(threshold, b, r, xq) * false_positive_weight
                   + _false_negative_probability(threshold, b, r, xq) * false_negative_weight)
            if err < best:
                best, opt = err, (b, r)
    return opt


# ---- partitioning of the set-size domain (lshensemble_partition.py) -------------------------------------------
def _interval_costs(sizes: np.ndarray, counts: np.ndarray) -> np.ndarray:
    """cost[l, u] = expected false positives when every set with size in [sizes[l], sizes[u]] is treated as
    having size sizes[u] (lshensemble_partition.py:54-92): sum_i (sizes[u] - sizes[i]) / sizes[u] * counts[i]."""
    n = len(sizes)
    cost = np.zeros((n, n))
    for u in range(n):
        top = float(sizes[u])
        for l in range(u + 1):
            cost[l, u] = np.sum((top - sizes[l:u + 1]) / top * counts[l:u + 1])
    return cost


def optimal_partitions(sizes, counts, num_part: int) -> List[Tuple[int, int]]:
    """Cut the ascending domain of set sizes into ``num_part`` contiguous intervals ``(lower, upper)`` (inclusive)
    minimising the summed interval cost; ties go to the smaller cut index, as in the reference
    (lshensemble_partition.py:95-196)."""
    sizes = np.asarray(sizes)
    counts = np.asarray(counts)
    n = len(sizes)
    if num_part < 2:
        return [(sizes[0], sizes[-1])]
    if num_part >= n:
        return [(x, x) for x in sizes]
    cost = _interval_costs(sizes, counts)
    last = n - 1
    if num_part == 2:
        tot = cost[0, :last] + cost[1:, last]                      # first interval ends at u1, second is the rest
        u = int(np.argmin(tot))                                    # first minimum = smallest u1
        return [(sizes[0], sizes[u]), (sizes[u + 1], sizes[-1])]
    # tab[p][u] (p = 2 .. num_part-1): cheapest cover of sizes[0..u] by p intervals; entries with u < p-1 stay 0,
    # exactly like the reference's zero-initialised matrix (lshensemble_partition.py:130-146)
    tab: Dict[int, np.ndarray] = {}
    for p in range(2, num_part):
        t = np.zeros(n)
        prev = cost[0] if p == 2 else tab[p - 1]
        for u in range(p - 1, n):
            t[u] = np.min(prev[p - 2:u] + cost[p - 1:u + 1, u])    # u1 = p-2 .. u-1, next interval = u1+1 .. u
        tab[p] = t
    p = num_part
    u = p - 2 + int(np.argmin(tab[p - 1][p - 2:last] + cost[p - 1:last + 1, last]))
    bounds = [(sizes[u + 1], sizes[-1])]
    p -= 1
    while p > 1:
        # NOTE: the reference's back-tracking reads the p-interval table here, where the recurrence that filled the
        # tables used p-1 (lshensemble_partition.py:158-166).  Reproduced as is: the partition bounds have to be the
        # reference's, not the optimum of the recurrence.
        u1 = p - 2 + int(np.argmin(tab[p][p - 2:u] + cost[p - 1:u + 1, u]))
        bounds.insert(0, (sizes[u1 + 1], sizes[u]))
        u = u1
        p -= 1
    bounds.insert(0, (sizes[0], sizes[u]))
    return bounds


def optimal_partitions_device(sizes, counts, num_part: int, device: int = 0) -> List[Tuple[int, int]]:
    """``optimal_partitions(sizes, counts, num_part)``, the same list of ``(lower, upper)`` tuples of the input's sizes, with
    the interval costs, the dynamic programme and the back-tracking on CUDA device ``device`` (``dsk_ensemble_partition``).

    ``sizes`` (strictly ascending, > 0) and ``counts`` (> 0) are integer sequences of one length D >= 1, each value below
    2^62; ``ValueError`` otherwise.  Every cost is the reference's float64 value bit for bit (its numpy pairwise sums
    included) and every argmin takes the first index among equal values, so the bounds are the reference's.  The
    workspace, about ``4 * D * (D + 1) + 8 * D * num_part`` bytes of device memory (``dsk_ensemble_partition_workspace_size``),
    is allocated with torch; ``MemoryError`` names D and the bytes if it cannot be.  ``num_part < 2`` and ``num_part >= D``
    need no table and are answered on the host, as in ``optimal_partitions``."""
    from . import _native as nv
    sz = np.asarray(sizes)
    ct = np.asarray(counts)
    if sz.ndim != 1 or ct.ndim != 1 or len(sz) != len(ct) or len(sz) == 0:
        raise ValueError("sizes and counts must be 1-D sequences of one length >= 1 (got %s and %s)" % (sz.shape, ct.shape))
    if sz.dtype.kind not in "iu" or ct.dtype.kind not in "iu":
        raise TypeError("set sizes and counts must be integers")
    if np.any(sz < 0) or np.any(ct < 0):   # a negative value would wrap in a uint64 -> int64 cast; the C-ABI names it
        raise ValueError("set sizes and counts must be positive")
    s64 = np.ascontiguousarray(sz, dtype=np.int64)
    c64 = np.ascontiguousarray(ct, dtype=np.int64)
    n = len(s64)
    lib = nv.load()
    out = np.zeros(max(min(num_part, n), 1), dtype=np.int64)
    if num_part < 2 or num_part >= n:   # no table: the C-ABI only checks the input and writes the trivial bounds
        nv.check(lib.dsk_ensemble_partition(s64.ctypes.data, c64.ctypes.data, n, num_part, None, 0, device,
                                            out.ctypes.data, None, None))
    else:
        import torch
        nv.require_device(device)
        need = int(lib.dsk_ensemble_partition_workspace_size(n, num_part))
        try:
            ws = torch.empty((need,), dtype=torch.uint8, device="cuda:%d" % device)
        except torch.OutOfMemoryError as exc:
            raise MemoryError("optimal_partitions_device: cannot allocate the %d bytes of device memory the partitioner "
                              "needs for D = %d distinct set sizes and num_part = %d" % (need, n, num_part)) from exc
        with torch.cuda.device(device):
            nv.check(lib.dsk_ensemble_partition(s64.ctypes.data, c64.ctypes.data, n, num_part, ws.data_ptr(), need, device,
                                                out.ctypes.data, None, torch.cuda.current_stream().cuda_stream))
        del ws
    if num_part < 2:
        return [(sz[0], sz[-1])]
    if num_part >= n:
        return [(x, x) for x in sz]
    lowers = np.concatenate([[0], out[:-1] + 1])
    return [(sz[lo], sz[up]) for lo, up in zip(lowers.tolist(), out.tolist())]


# ---- the index ------------------------------------------------------------------------------------------------
def _check_args(threshold, num_perm, num_part, m, weights) -> None:
    """The constructor's argument checks (lshensemble.py:120-133)."""
    if threshold > 1.0 or threshold < 0.0:
        raise ValueError("threshold must be in [0.0, 1.0]")
    if num_perm < 2:
        raise ValueError("Too few permutation functions")
    if num_part < 1:
        raise ValueError("num_part must be at least 1")
    if m < 2 or m > num_perm:
        raise ValueError("m must be in the range of [2, num_perm]")
    if any(w < 0.0 or w > 1.0 for w in weights):
        raise ValueError("Weight must be in [0.0, 1.0]")
    if sum(weights) != 1.0:
        raise ValueError("Weights must sum to 1.0")


class MinHashLSHEnsemble:
    """LSH Ensemble for containment queries (constructor contract of lshensemble.py:108-153)."""

    def __init__(self, threshold: float = 0.9, num_perm: int = 128, num_part: int = 16, m: int = 8,
                 weights: Tuple[float, float] = (0.5, 0.5), storage_config: Optional[dict] = None,
                 prepickle: Optional[bool] = None) -> None:
        _check_args(threshold, num_perm, num_part, m, weights)
        self.threshold = threshold
        self.h = num_perm
        self.m = m
        rs = self._init_optimal_params(weights)
        storage_config = storage_config if storage_config else {"type": "dict"}
        basename = storage_config.get("basename", _random_name(11))
        self.indexes = [
            {r: MinHashLSH(num_perm=self.h, params=(int(self.h / r), r),
                           storage_config=self._get_storage_config(basename, storage_config, part, r),
                           prepickle=prepickle) for r in rs}
            for part in range(num_part)]
        self.lowers = [None for _ in self.indexes]
        self.uppers = [None for _ in self.indexes]

    def _init_optimal_params(self, weights):
        fpw, fnw = weights
        self.xqs = np.exp(np.linspace(-5, 5, 10))
        self.params = np.array([_optimal_param(self.threshold, self.h, self.m, xq, fpw, fnw) for xq in self.xqs],
                               dtype=int)
        return {r for _, r in self.params}

    def _get_optimal_param(self, x, q):
        i = np.searchsorted(self.xqs, float(x) / float(q), side="left")
        if i == len(self.params):
            i -= 1
        return self.params[i]

    def _get_storage_config(self, basename, base_config, partition, r):
        config = dict(base_config)
        config["basename"] = b"-".join([basename, struct.pack(">H", partition), struct.pack(">H", r)])
        return config

    def index(self, entries: Iterable[Tuple[Hashable, MinHash, int]]) -> None:
        """Index all sets given as ``(key, minhash, size)``; callable once (lshensemble.py:189-228)."""
        if not self.is_empty():
            raise ValueError("Cannot call index again on a non-empty index")
        if not isinstance(entries, list):
            checked = []
            for key, minhash, size in entries:
                if size <= 0:
                    raise ValueError("Set size must be positive")
                checked.append((key, minhash, size))
            entries = checked
        if len(entries) == 0:
            raise ValueError("entries is empty")
        sizes, counts = np.array(sorted(Counter(e[2] for e in entries).most_common())).T
        partitions = optimal_partitions(sizes, counts, len(self.indexes))
        for i, (lower, upper) in enumerate(partitions):
            self.lowers[i], self.uppers[i] = lower, upper
        entries.sort(key=lambda e: e[2])
        # same walk as the reference (one step to the next partition when a size exceeds the current upper bound),
        # but the partition's sets are inserted together so their band keys come from one kernel launch per r
        groups: List[list] = [[] for _ in self.indexes]
        curr = 0
        for e in entries:
            if e[2] > self.uppers[curr]:
                curr += 1
            groups[curr].append(e)
        for part, members in enumerate(groups):
            if not members:
                continue
            keys = [e[0] for e in members]
            mhs = [e[1] for e in members]
            batchable = all(np.ndim(mh.hashvalues) == 1 for mh in mhs)
            for r, lsh in self.indexes[part].items():
                if batchable:
                    lsh.insert_batch(keys, mhs)
                else:  # WeightedMinHash rows are (k, t) pairs: per-object path
                    for k, mh in zip(keys, mhs):
                        lsh.insert(k, mh)

    def query(self, minhash, size: int) -> Generator[Hashable, None, None]:
        """Keys of sets whose containment of the query exceeds the threshold (lshensemble.py:230-249)."""
        for i, index in enumerate(self.indexes):
            u = self.uppers[i]
            if u is None:
                continue
            b, r = self._get_optimal_param(u, size)
            for key in index[r]._query_b(minhash, b):
                yield key

    def __contains__(self, key: Hashable) -> bool:
        return any(any(key in index[r] for r in index) for index in self.indexes)

    def is_empty(self) -> bool:
        return all(all(index[r].is_empty() for r in index) for index in self.indexes)


# ---- device-resident index ------------------------------------------------------------------------------------
def _partition_ranges(sorted_sizes: np.ndarray, uppers: list) -> np.ndarray:
    """``start[0..num_part]``: the reference's walk over the size-sorted sets (lshensemble.py:216-228) -- a set whose size
    exceeds the current partition's upper bound moves the walk ONE partition on -- as ranges of sorted set numbers.
    Equal sizes form a run; inside a run the walk can only move while the size exceeds the current bound, so each run is
    handled in a few steps."""
    n_part = len(uppers)
    start = np.zeros(n_part + 1, dtype=np.int64)
    vals, first = np.unique(sorted_sizes, return_index=True)
    ends = np.append(first[1:], len(sorted_sizes))
    curr = 0
    for v, a, e in zip(vals.tolist(), first.tolist(), ends.tolist()):
        while a < e and v > uppers[curr]:   # this set opens the next partition
            curr += 1
            start[curr] = a
            a += 1
    start[curr + 1:] = len(sorted_sizes)
    return start


def _index_plan(sizes: np.ndarray, num_part: int, partitioner=optimal_partitions):
    """Plan of ``GpuLSHEnsemble.index`` for set sizes ``int64[N]``: ``(lowers, uppers, order, start)`` -- the
    reference's partition bounds over ``Counter(sizes)`` (None for the unused trailing partitions) from ``partitioner``
    (``optimal_partitions`` or a function with its contract, such as ``optimal_partitions_device`` bound to a device),
    the stable size order (``order[t]`` = the row that becomes set number t, as ``entries.sort(key=size)``) and the
    partitions as ranges of set numbers."""
    vals, counts = np.unique(sizes, return_counts=True)      # = sorted(Counter(sizes).most_common())
    lowers, uppers = [None] * num_part, [None] * num_part
    for i, (lower, upper) in enumerate(partitioner(vals, counts, num_part)):
        lowers[i], uppers[i] = lower, upper
    order = np.argsort(sizes, kind="stable")
    return lowers, uppers, order, _partition_ranges(sizes[order], uppers)


def _selection(xqs: np.ndarray, n_params: int, uppers: list, start: np.ndarray, sizes) -> np.ndarray:
    """``int32[Q, num_part]``: the row of the (b, r) table each query uses in each partition -- ``_get_optimal_param(upper,
    size)``'s ``searchsorted(xqs, float(upper) / float(size), side="left")`` clamped to the last row, in float64 as
    there -- or -1 where the partition has no upper bound or no sets."""
    sizes = np.asarray(sizes, dtype=np.int64).reshape(-1)
    sel = np.full((len(sizes), len(uppers)), -1, dtype=np.int32)
    for p, u in enumerate(uppers):
        if u is None or start[p] == start[p + 1]:
            continue
        i = np.searchsorted(xqs, float(u) / sizes.astype(np.float64), side="left")
        sel[:, p] = np.minimum(i, n_params - 1)
    return sel


class GpuLSHEnsemble:
    """Device-resident ``MinHashLSHEnsemble``: containment search ("which indexed sets contain most of this query set")
    over whole signature matrices.

    The constructor's arguments, checks, ``params`` / ``xqs`` (the (b, r) table) and, after ``index``, ``lowers`` /
    ``uppers`` (the size partitions) are the host class's.  ``index(sig, sizes)`` takes the N sets as the rows of a
    signature matrix; ``query(sig, sizes)`` returns CSR arrays ``(ptr, idx)`` whose ``idx[ptr[q]:ptr[q+1]]`` are, as a
    set, ``MinHashLSHEnsemble.query(m_q, size_q)`` on the same data, given as row numbers of the ``index`` call.

    On the device the rows are held once, in size order, so each partition is a range of set numbers; for each distinct r
    of the table one set of ``num_perm // r`` band tables is keyed by (partition, band, r-tuple).  Device memory, in
    bytes, with ``cap`` the power of two >= 2N: ``4*K*N + 4*N + sum over distinct r of (K // r) * (16*cap + 4*N)``
    (``dsk_lsh_ensemble_index_bytes``)."""

    def __init__(self, threshold: float = 0.9, num_perm: int = 128, num_part: int = 16, m: int = 8,
                 weights: Tuple[float, float] = (0.5, 0.5), device: int = 0) -> None:
        _check_args(threshold, num_perm, num_part, m, weights)
        self.threshold = threshold
        self.h = num_perm
        self.m = m
        self.num_part = num_part
        self.device = device
        MinHashLSHEnsemble._init_optimal_params(self, weights)   # self.xqs, self.params
        self.lowers: list = [None] * num_part
        self.uppers: list = [None] * num_part
        self.keys: Optional[list] = None
        self._keyset: Optional[set] = None
        self._start = np.zeros(num_part + 1, dtype=np.int64)
        self._set_sizes: Optional[np.ndarray] = None   # int64[N] of the index call, in its row order
        self._d_set_sizes = None                        # their device copy, made by the first call that needs it
        from . import _native as nv
        nv.require_device(device)
        b = np.ascontiguousarray(self.params[:, 0], dtype=np.int32)
        r = np.ascontiguousarray(self.params[:, 1], dtype=np.int32)
        h = ctypes.c_void_p()
        nv.check(nv.load().dsk_lsh_ensemble_create(num_perm, num_part, b.ctypes.data, r.ctypes.data, len(b), device,
                                                   ctypes.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                from . import _native as nv
                nv.load().dsk_lsh_ensemble_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass

    _get_optimal_param = MinHashLSHEnsemble._get_optimal_param

    def __len__(self) -> int:
        from . import _native as nv
        n = ctypes.c_int64()
        nv.check(nv.load().dsk_lsh_ensemble_size(self._h, ctypes.byref(n)))
        return int(n.value)

    def is_empty(self) -> bool:
        return len(self) == 0

    def __contains__(self, key: Hashable) -> bool:
        if self._keyset is not None:
            return key in self._keyset
        return isinstance(key, (int, np.integer)) and 0 <= key < len(self)

    def _dev_sig(self, sig):
        import torch
        from .lsh import _signature_matrix
        if isinstance(sig, np.ndarray):
            sig = torch.from_numpy(_signature_matrix(sig).view(np.int32)).cuda(self.device)
        if sig.dim() != 2 or sig.shape[1] != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, sig.shape[-1]))
        if sig.element_size() != 4:
            raise TypeError("GpuLSHEnsemble takes the 32-bit signature matrix")
        return sig.contiguous()

    @staticmethod
    def _sizes(sizes, n: int) -> np.ndarray:
        s = np.asarray(sizes.cpu() if hasattr(sizes, "cpu") else sizes).reshape(-1)
        if s.size and s.dtype.kind not in "iu":
            raise TypeError("set sizes must be integers")
        s = s.astype(np.int64)
        if len(s) != n:
            raise ValueError("sizes must hold one size per row of sig (%d), got %d" % (n, len(s)))
        return s

    def index(self, sig, sizes, keys: Optional[Iterable[Hashable]] = None) -> None:
        """Index the N sets given as the rows of ``sig`` ([N, K] uint32; numpy or CUDA tensor) with their sizes
        (``int64[N]``, each > 0) and, optionally, one key per row.  Callable once, like the reference's ``index``; set j
        is row j of this call.  Raises ``ValueError`` as the reference does for a second call, no sets and a size <= 0,
        and for mismatched lengths or a wrong K; ``MemoryError`` if the device memory cannot be allocated, after which
        the object is still empty and can index."""
        import torch
        from . import _native as nv
        if not self.is_empty():
            raise ValueError("Cannot call index again on a non-empty index")
        n = int(sig.shape[0]) if sig.ndim == 2 else -1
        if n == 0:
            raise ValueError("entries is empty")
        d_sig = self._dev_sig(sig)
        sizes = self._sizes(sizes, n)
        if np.any(sizes <= 0):
            raise ValueError("Set size must be positive")
        if keys is not None:
            keys = list(keys)
            if len(keys) != n:
                raise ValueError("keys must hold one key per row of sig (%d), got %d" % (n, len(keys)))
        if n >= 1 << 31:
            raise ValueError("an index holds fewer than 2^31 sets")
        lowers, uppers, order, start = _index_plan(
            sizes, self.num_part, lambda s, c, k: optimal_partitions_device(s, c, k, device=self.device))
        d_order = torch.from_numpy(order.astype(np.int32)).to(d_sig.device)
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_lsh_ensemble_index(self._h, d_sig.data_ptr(), n, d_order.data_ptr(), start.ctypes.data,
                                                      torch.cuda.current_stream().cuda_stream))
        self.lowers, self.uppers, self._start = lowers, uppers, start
        self._set_sizes, self._d_set_sizes = sizes, None
        if keys is not None:
            self.keys, self._keyset = keys, set(keys)

    def selection(self, sizes) -> np.ndarray:
        """``int32[Q, num_part]``: the row of ``params`` each query size uses in each partition (``_get_optimal_param``),
        -1 where the partition has no upper bound or no sets."""
        return _selection(self.xqs, len(self.params), self.uppers, self._start, sizes)

    def query(self, sig, sizes, with_eq: bool = False, to_host: bool = True):
        """Containment candidates of every row of ``sig`` with its set size (each > 0): ``(ptr int64[Q+1], idx
        int32[M])``, plus ``eq int32[M]`` when ``with_eq``.

        ``idx[ptr[q]:ptr[q+1]]`` lists each candidate once, unordered, as a row number of the ``index`` call; as a set it is
        ``MinHashLSHEnsemble.query(m_q, size_q)``: over every partition p with an upper bound, with ``(b, r) =
        params[selection(size_q)[p]]``, the sets of p that share the query's r-tuple in one of the first b bands of the
        ``(num_perm // r, r)`` banding.  ``eq`` is the number of the ``num_perm`` positions where the query row and the
        candidate's row agree (``eq / num_perm`` is ``MinHash.jaccard``): with the two sizes it estimates containment."""
        import torch
        from . import _native as nv
        d_q = self._dev_sig(sig)
        nq = int(d_q.shape[0])
        sizes = self._sizes(sizes, nq)
        if np.any(sizes <= 0):
            raise ValueError("Set size must be positive")
        dev = d_q.device
        lib = nv.load()
        items = nq * self.num_part
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            sel = torch.from_numpy(self.selection(sizes)).to(dev)
            counts = torch.empty((max(items, 1),), dtype=torch.int64, device=dev)
            iptr = torch.empty((items + 1,), dtype=torch.int64, device=dev)
            scratch = torch.empty((items // 1024 + 2,), dtype=torch.int64, device=dev)
            nv.check(lib.dsk_lsh_ensemble_query_count(self._h, d_q.data_ptr(), nq, sel.data_ptr(), counts.data_ptr(), st))
            nv.check(lib.dsk_exclusive_scan(counts.data_ptr(), items, iptr.data_ptr(), scratch.data_ptr(), st))
            total = int(iptr[items].item())
            idx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            eq = torch.empty((max(total, 1),), dtype=torch.int32, device=dev) if with_eq else None
            nv.check(lib.dsk_lsh_ensemble_query_fill(self._h, d_q.data_ptr(), nq, sel.data_ptr(), iptr.data_ptr(),
                                                     idx.data_ptr(), eq.data_ptr() if with_eq else None, st))
            ptr = iptr[::self.num_part].contiguous()
            out = (ptr, idx[:total]) + ((eq[:total],) if with_eq else ())
        if to_host:
            return tuple(x.cpu().numpy() for x in out)
        return out

    def query_keys(self, sig, sizes) -> List[list]:
        """Like ``GpuLSH.query_keys``: per query, the list of keys (or row numbers, without keys) of its candidates."""
        ptr, idx = self.query(sig, sizes)
        out = []
        for q in range(len(ptr) - 1):
            ids = idx[ptr[q]:ptr[q + 1]]
            out.append([self.keys[i] for i in ids] if self.keys is not None else ids.tolist())
        return out

    # -- containment estimates on the device -----------------------------------------------------------------------
    def _containment_args(self, sig, sizes, min_containment):
        """The query matrix, its sizes (host and device), the device copy of the indexed sizes (a placeholder before
        ``index``: nothing reads it) and the threshold as a float.  Query sizes must be in [1, 2^62) so that s_q + s_x
        fits in int64."""
        import torch
        d_q = self._dev_sig(sig)
        sizes = self._sizes(sizes, int(d_q.shape[0]))
        if np.any(sizes <= 0) or np.any(sizes >= 1 << 62):
            raise ValueError("query set sizes must be in [1, 2^62)")
        d_xs = self._device_set_sizes()
        if d_xs is None:
            d_xs = torch.zeros((1,), dtype=torch.int64, device=d_q.device)
        return d_q, sizes, torch.from_numpy(sizes).to(d_q.device), d_xs, _min_containment(min_containment)

    def _device_set_sizes(self):
        import torch
        if self._d_set_sizes is None and self._set_sizes is not None:
            self._d_set_sizes = torch.from_numpy(self._set_sizes).cuda(self.device)
        return self._d_set_sizes

    def _containment_csr(self, count, fill, items: int, dev, to_host: bool):
        """count(counts) / dsk_exclusive_scan / fill(iptr, idx, eq, c) over ``items`` (query, partition) items, as ``query``;
        returns ``(ptr, idx, eq, containment)`` with ptr over the items' queries."""
        import torch
        from . import _native as nv
        counts = torch.empty((max(items, 1),), dtype=torch.int64, device=dev)
        iptr = torch.empty((items + 1,), dtype=torch.int64, device=dev)
        scratch = torch.empty((items // 1024 + 2,), dtype=torch.int64, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        nv.check(count(counts.data_ptr(), st))
        nv.check(nv.load().dsk_exclusive_scan(counts.data_ptr(), items, iptr.data_ptr(), scratch.data_ptr(), st))
        total = int(iptr[items].item())
        idx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
        eq = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
        c = torch.empty((max(total, 1),), dtype=torch.float64, device=dev)
        nv.check(fill(iptr.data_ptr(), idx.data_ptr(), eq.data_ptr(), c.data_ptr(), st))
        out = (iptr[::self.num_part].contiguous(), idx[:total], eq[:total], c[:total])
        return tuple(x.cpu().numpy() for x in out) if to_host else out

    def query_containment(self, sig, sizes, min_containment: Optional[float] = None, to_host: bool = True):
        """``query(sig, sizes, with_eq=True)`` with the containment estimate of each candidate, filtered on the device:
        ``(ptr int64[Q+1], idx int32[M], eq int32[M], containment float64[M])``, each kept candidate once, unordered.

        For query q of size s_q and candidate x of size s_x (its size in the ``index`` call), with ``j = eq / num_perm``
        (``MinHash.jaccard``), ``c = j * (s_q + s_x) / (s_q * (1 + j))``: the inverse of the map t -> t / (1 + s_x/s_q - t)
        that the (b, r) table was chosen with, so c estimates |Q & X| / |Q|.  It is the float64 value of that Python
        expression bit for bit, and it is not clamped: with s_x > s_q and j near 1 it exceeds 1 (``min(c, 1.0)`` caps it).
        A candidate is kept iff ``c >= min_containment``: ``[x for x in ens.query(m, s) if c(m, s, x) >= t]``.
        ``min_containment`` is None (keep all, the same as 0.0) or a float in [0, 1]; query sizes are in [1, 2^62);
        ``ValueError`` otherwise."""
        import torch
        from . import _native as nv
        d_q, sizes, d_qs, d_xs, t = self._containment_args(sig, sizes, min_containment)
        nq = len(sizes)
        lib = nv.load()
        with torch.cuda.device(self.device):
            sel = torch.from_numpy(self.selection(sizes)).to(d_q.device)
            args = (self._h, d_q.data_ptr(), nq, d_qs.data_ptr(), sel.data_ptr(), d_xs.data_ptr(), t)
            return self._containment_csr(
                lambda counts, st: lib.dsk_lsh_ensemble_containment_count(*args, counts, st),
                lambda iptr, idx, eq, c, st: lib.dsk_lsh_ensemble_containment_fill(*args, iptr, idx, eq, c, st),
                nq * self.num_part, d_q.device, to_host)

    def query_topk(self, sig, sizes, k: int, min_containment: Optional[float] = None, to_host: bool = True):
        """Each query's k (1..32) kept candidates of largest containment estimate: ``(idx int32[Q, k], eq int32[Q, k],
        containment float64[Q, k])``, in the order ``sorted(kept, key=lambda x: (-c, x))[:k]`` (ties to the smaller row of
        the ``index`` call), padded with -1 / -1 / -1.0.  Candidates, estimate and filter are ``query_containment``'s.  One
        kernel launch after the selection table and the sizes are uploaded."""
        import torch
        from . import _native as nv
        from .lsh import _check_topk
        k = _check_topk(k)
        d_q, sizes, d_qs, d_xs, t = self._containment_args(sig, sizes, min_containment)
        nq = len(sizes)
        dev = d_q.device
        with torch.cuda.device(self.device):
            sel = torch.from_numpy(self.selection(sizes)).to(dev)
            idx = torch.empty((nq, k), dtype=torch.int32, device=dev)
            eq = torch.empty((nq, k), dtype=torch.int32, device=dev)
            c = torch.empty((nq, k), dtype=torch.float64, device=dev)
            nv.check(nv.load().dsk_lsh_ensemble_containment_topk(
                self._h, d_q.data_ptr(), nq, d_qs.data_ptr(), sel.data_ptr(), d_xs.data_ptr(), t, k, idx.data_ptr(),
                eq.data_ptr(), c.data_ptr(), torch.cuda.current_stream().cuda_stream))
        out = (idx, eq, c)
        return tuple(x.cpu().numpy() for x in out) if to_host else out

    def containment_pairs(self, min_containment: Optional[float] = None, to_host: bool = True):
        """The self-join: CSR ``(ptr int64[N+1], idx, eq, containment)`` over the rows of the ``index`` call, row i being
        ``query_containment`` of indexed row i with its own size, without i itself -- the sets that contain at least
        ``min_containment`` of set i (by the estimate).  Set i is left out by identity: an equal row of equal size is
        listed.  It reads the index's own rows, so no copy of the signatures is needed.  An index never built gives
        ``ptr = [0]``."""
        import torch
        from . import _native as nv
        t = _min_containment(min_containment)
        dev = torch.device("cuda", self.device)
        if self._set_sizes is None:
            out = (torch.zeros((1,), dtype=torch.int64, device=dev), torch.zeros((0,), dtype=torch.int32, device=dev),
                   torch.zeros((0,), dtype=torch.int32, device=dev), torch.zeros((0,), dtype=torch.float64, device=dev))
            return tuple(x.cpu().numpy() for x in out) if to_host else out
        lib = nv.load()
        with torch.cuda.device(self.device):
            d_xs = self._device_set_sizes()
            sel = torch.from_numpy(self.selection(self._set_sizes)).to(dev)
            args = (self._h, sel.data_ptr(), d_xs.data_ptr(), t)
            return self._containment_csr(
                lambda counts, st: lib.dsk_lsh_ensemble_self_containment_count(*args, counts, st),
                lambda iptr, idx, eq, c, st: lib.dsk_lsh_ensemble_self_containment_fill(*args, iptr, idx, eq, c, st),
                len(self._set_sizes) * self.num_part, dev, to_host)


def _min_containment(t) -> float:
    """``min_containment``: None -> 0.0 (every candidate, c >= 0), else a float in [0, 1]; ``ValueError`` otherwise
    (NaN included)."""
    if t is None:
        return 0.0
    if isinstance(t, bool) or not isinstance(t, (int, float, np.integer, np.floating)):
        raise ValueError("min_containment must be None or a float in [0.0, 1.0], got %r" % (t,))
    t = float(t)
    if not 0.0 <= t <= 1.0:
        raise ValueError("min_containment must be in [0.0, 1.0], got %r" % (t,))
    return t
