"""Weighted MinHash with the reference's API (datasketch/weighted_minhash.py:11-159).

``WeightedMinHashGenerator.__init__`` draws the ICWS parameters on the host with numpy,
bit-identically to the reference (:118-121).  ``minhash`` (one vector) and
``minhash_batch`` (a matrix) run the per-sample argmin in ``libdsk_b200.so``
(``dsk_wmh_minhash``); every float32 step after ``log`` is IEEE-identical to numpy.  Sparse matrices
(scipy.sparse, CUDA ``torch.sparse_csr``) go to ``dsk_wmh_minhash_csr`` as their stored entries, with the results of
their densified rows.
"""
from __future__ import annotations

import collections.abc
import copy
import ctypes
from typing import List, Optional

import numpy as np

from . import _native as nv


class WeightedMinHash:
    """Container produced by :class:`WeightedMinHashGenerator` (weighted_minhash.py:11-95)."""

    def __init__(self, seed: int, hashvalues: np.ndarray) -> None:
        self.seed = seed
        self.hashvalues = hashvalues

    def jaccard(self, other: "WeightedMinHash") -> float:
        """Fraction of samples whose (k, t) rows agree (weighted_minhash.py:28-60)."""
        if other.seed != self.seed:
            raise ValueError("Cannot compute Jaccard given WeightedMinHash objects with different seeds")
        if len(self) != len(other):
            raise ValueError("Cannot compute Jaccard given WeightedMinHash objects with different numbers of "
                             "hash values")
        same = np.all(np.asarray(self.hashvalues) == np.asarray(other.hashvalues), axis=1)
        return float(np.count_nonzero(same)) / float(len(self))

    def digest(self) -> np.ndarray:
        return copy.copy(self.hashvalues)

    def copy(self) -> "WeightedMinHash":
        return WeightedMinHash(self.seed, self.digest())

    def __len__(self) -> int:
        return len(self.hashvalues)

    def __eq__(self, other) -> bool:
        return (type(self) is type(other) and self.seed == other.seed
                and np.array_equal(self.hashvalues, other.hashvalues))

    __hash__ = None


def _is_sparse(X) -> bool:
    """A scipy.sparse matrix or array, or a torch tensor in the sparse CSR layout."""
    if hasattr(X, "tocsr") and hasattr(X, "nnz"):
        return True
    layout = getattr(X, "layout", None)
    return layout is not None and str(layout) == "torch.sparse_csr"


def _csr_arrays(X, dim: int):
    """A scipy.sparse matrix -> (indptr int64 [n + 1], indices int32 [nnz], weights float32 [nnz]) in canonical CSR
    form, whose rows densify to exactly ``np.asarray(X.tocsr().toarray(), dtype=np.float32)``.

    ``toarray()`` sums duplicate entries in the matrix's own dtype, in stored order, starting from 0; in float32
    ``1 + 1e8 - 1e8`` is 0 but ``1e8 - 1e8 + 1`` is 1, so the order matters.  A stable sort by column within each row
    keeps that order and ``np.add.at`` adds in it (``sum_duplicates()`` sorts unstably).  The cast to float32 follows
    the sums, as it follows ``toarray()``."""
    X = X.tocsr()
    if X.ndim != 2 or X.shape[1] != dim:
        raise ValueError("Input dimension mismatch, expecting %d" % dim)
    n = X.shape[0]
    indptr = np.asarray(X.indptr, dtype=np.int64)
    indices, data = np.asarray(X.indices), np.asarray(X.data)
    if (len(indptr) != n + 1 or indptr[0] != 0 or bool((indptr[1:] < indptr[:-1]).any())
            or indptr[-1] > min(len(indices), len(data))):
        raise ValueError("the matrix's indptr must start at 0, be non-decreasing and end at most at nnz")
    nnz = int(indptr[-1])
    indices, data = indices[:nnz], data[:nnz]
    if nnz and (int(indices.min()) < 0 or int(indices.max()) >= dim):
        bad = (indices < 0) | (indices >= dim)
        raise ValueError("row %d: column indices fall outside [0, %d)"
                         % (int(np.searchsorted(indptr, np.argmax(bad), side="right")) - 1, dim))
    if not X.has_canonical_format:
        key = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr)) * dim + indices.astype(np.int64)
        order = np.argsort(key, kind="stable")
        key = key[order]
        first = np.ones(len(key), dtype=bool)
        first[1:] = key[1:] != key[:-1]
        summed = np.zeros(int(first.sum()), dtype=data.dtype)
        np.add.at(summed, np.cumsum(first) - 1, data[order])
        key, data = key[first], summed
        indices = key % dim
        indptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(key // dim, minlength=n), out=indptr[1:])
    return indptr, indices.astype(np.int32, copy=False), data.astype(np.float32, copy=False)


class WeightedMinHashGenerator:
    """Creates :class:`WeightedMinHash` objects (weighted_minhash.py:98-159)."""

    def __init__(self, dim: int, sample_size: int = 128, seed: int = 1) -> None:
        self.dim = dim
        self.sample_size = sample_size
        self.seed = seed
        generator = np.random.RandomState(seed=seed)
        # drawn in exactly this order from one RandomState (weighted_minhash.py:118-121)
        self.rs = generator.gamma(2, 1, (sample_size, dim)).astype(np.float32)
        self.ln_cs = np.log(generator.gamma(2, 1, (sample_size, dim))).astype(np.float32)
        self.betas = generator.uniform(0, 1, (sample_size, dim)).astype(np.float32)
        self._handles = {}

    # -- device state (dropped on pickling) -----------------------------------------------------
    def _handle(self, device: int = 0):
        h = self._handles.get(device)
        if h is None:
            nv.require_device(device)
            ptr = ctypes.c_void_p()
            rs, lc, be = (np.ascontiguousarray(x, dtype=np.float32) for x in (self.rs, self.ln_cs, self.betas))
            nv.check(nv.load().dsk_wmh_create(rs.ctypes.data, lc.ctypes.data, be.ctypes.data, self.sample_size,
                                              self.dim, device, ctypes.byref(ptr)))
            h = ptr
            self._handles[device] = h
        return h

    def __del__(self):
        try:
            for h in getattr(self, "_handles", {}).values():
                nv.load().dsk_wmh_destroy(h)
            self._handles = {}
        except Exception:  # noqa: BLE001
            pass

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_handles"] = {}
        return st

    # -- sampling ----------------------------------------------------------------------------------
    def _sample(self, X, device: int, many: bool, device_log: bool = False, to_host: bool = True):
        """Device pass over [n, dim] weights -> ([n, sample_size, 2] int64 of (k, t), [n] int32 status), as numpy
        arrays or (``to_host=False``) as the CUDA tensors the kernel wrote.  Status 1 marks a row with no candidate
        column (all zeros; for ``many=False`` also all negative or NaN), status 2 a row whose t is not finite (a +inf
        weight; stored as INT64_MIN).

        For numpy input the logarithm is taken on the HOST with numpy's own float32 ``log`` -- the very call the
        reference makes (weighted_minhash.py:150-152, ``vlog = np.log(v)``; zeros give -inf here and are skipped) --
        and the kernel gets ``vlog`` (``DSK_WMH_INPUT_LOG``), so every step is bit-identical to the reference by
        construction.  ``device_log=True`` (and CUDA tensor input) lets the kernel take the logarithm itself: one
        pass less over the data.  Its log is the float64 log rounded to float32, which is not always numpy's (numpy's
        float32 log can be up to 3 ulp from the correctly rounded one), so (k, t) can differ from the reference's on
        float near-ties."""
        import torch
        flags = int(many)
        if isinstance(X, np.ndarray):
            X = np.ascontiguousarray(X, dtype=np.float32)
            if X.ndim != 2 or X.shape[1] != self.dim:
                raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
            h = self._handle(device)
            if not device_log:
                with np.errstate(invalid="ignore", divide="ignore"):
                    X = np.log(X)
                flags |= 2   # DSK_WMH_INPUT_LOG
            d_v = torch.from_numpy(X).cuda(device)
        else:
            if X.dim() != 2 or X.shape[1] != self.dim:
                raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
            d_v = X.to(dtype=torch.float32).contiguous()
            device = d_v.device.index
            h = self._handle(device)
        n = d_v.shape[0]
        d_out = torch.empty((n, self.sample_size, 2), dtype=torch.int64, device=d_v.device)
        d_st = torch.empty((n,), dtype=torch.int32, device=d_v.device)
        with torch.cuda.device(device):
            nv.check(nv.load().dsk_wmh_minhash(h, d_v.data_ptr(), n, d_out.data_ptr(), d_st.data_ptr(), flags,
                                               torch.cuda.current_stream(d_v.device).cuda_stream))
        if not to_host:
            return d_out, d_st
        return d_out.cpu().numpy(), d_st.cpu().numpy()

    def _sample_csr(self, X, device: int, many: bool, device_log: bool = False, to_host: bool = True):
        """``_sample`` for sparse rows through ``dsk_wmh_minhash_csr``: a scipy.sparse matrix (prepared on the host by
        :func:`_csr_arrays`; host logarithm unless ``device_log``) or a CUDA ``torch.sparse_csr`` tensor (device
        logarithm).  Status 3 marks a row whose columns are not strictly increasing or fall outside [0, dim)."""
        import torch
        flags = int(many)
        if isinstance(X, torch.Tensor):
            if X.dim() != 2 or X.shape[1] != self.dim:
                raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
            if not X.is_cuda:
                raise ValueError("a torch.sparse_csr input must be a CUDA tensor")
            dev = X.device
            n = X.shape[0]
            indptr = X.crow_indices().to(torch.int64)
            cols = X.col_indices()
            if len(indptr) != n + 1 or bool(((indptr[0] != 0) | (indptr[-1] > len(cols))
                                             | (indptr[1:] < indptr[:-1]).any()).item()):
                raise ValueError("crow_indices must start at 0, be non-decreasing and end at most at nnz")
            # out-of-range columns become -1 or dim, which the kernel reports as status 3 (a plain int32 cast could wrap)
            cols = cols.clamp(-1, self.dim).to(torch.int32).contiguous()
            vals = X.values().to(torch.float32).contiguous()
        else:
            indptr, cols, vals = _csr_arrays(X, self.dim)
            n = len(indptr) - 1
            if not device_log:
                with np.errstate(invalid="ignore", divide="ignore"):
                    vals = np.log(vals)      # numpy's float32 log of the stored values, as the dense path takes it
                flags |= 2   # DSK_WMH_INPUT_LOG
            dev = torch.device("cuda", device)
            indptr, cols, vals = (torch.from_numpy(a).to(dev) for a in (indptr, cols, vals))
        if len(cols) == 0:                   # the kernel reads no entry, but its buffers must not be NULL
            cols = torch.zeros(1, dtype=torch.int32, device=dev)
            vals = torch.zeros(1, dtype=torch.float32, device=dev)
        h = self._handle(dev.index)
        d_out = torch.empty((n, self.sample_size, 2), dtype=torch.int64, device=dev)
        d_st = torch.empty((n,), dtype=torch.int32, device=dev)
        if n:
            with torch.cuda.device(dev):
                nv.check(nv.load().dsk_wmh_minhash_csr(h, indptr.data_ptr(), cols.data_ptr(), vals.data_ptr(), n,
                                                       d_out.data_ptr(), d_st.data_ptr(), flags,
                                                       torch.cuda.current_stream(dev).cuda_stream))
        bad = d_st == 3
        if n and bool(bad.any()):
            raise ValueError("row %d: column indices are not strictly increasing or fall outside [0, %d)"
                             % (int(bad.nonzero()[0][0]), self.dim))
        if not to_host:
            return d_out, d_st
        return d_out.cpu().numpy(), d_st.cpu().numpy()

    @staticmethod
    def _raise_status(status, empty_message: str) -> None:
        worst = int(status.max()) if len(status) else 0
        if worst and bool((status == 1).any()):
            raise ValueError(empty_message)
        if worst:
            raise OverflowError("cannot convert float infinity to integer")   # the reference's int(t[k]) (:158)

    def minhash_batch(self, X, device: int = 0, device_log: bool = False, to_host: bool = True):
        """[n, dim] weights -> [n, sample_size, 2] int64 of (k, t) -- row i equals
        ``self.minhash(X[i]).hashvalues``.  Raises ValueError if a row has no positive weight and OverflowError if
        one holds +inf.  ``to_host=False`` returns the CUDA int64 tensor (the same values), which
        ``GpuLSH(weighted=True)`` takes as it is: weights -> signatures -> index without a copy to the host.

        ``X`` may be sparse: a scipy.sparse matrix (row i equals ``minhash(X[i].toarray().ravel())``, with the host
        logarithm) or a CUDA ``torch.sparse_csr`` tensor (equal to ``minhash_batch(X.to_dense())``, with the device
        logarithm).  Sparse rows are sampled over their stored entries only, never densified."""
        if _is_sparse(X):
            out, status = self._sample_csr(X, device, many=False, device_log=device_log, to_host=to_host)
        else:
            out, status = self._sample(X, device, many=False, device_log=device_log, to_host=to_host)
        self._raise_status(status, "Input is all zeros")
        return out

    def minhash(self, v) -> WeightedMinHash:
        """One weighted Jaccard vector -> WeightedMinHash (weighted_minhash.py:123-159; same checks and errors:
        ValueError for an all-zero vector or one without a positive weight, OverflowError for a +inf weight)."""
        if not isinstance(v, collections.abc.Sized):
            raise TypeError("Input vector must be sized")
        if not len(v) == self.dim:
            raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
        v = np.array(v, dtype=np.float32)  # a private float32 copy: the input is never mutated
        if not (v != 0).any():
            raise ValueError("Input is all zeros")
        out, status = self._sample(v.reshape(1, -1), 0, many=False)
        self._raise_status(status, "All-NaN slice encountered")   # np.nanargmin's error (:157)
        return WeightedMinHash(self.seed, out[0].astype(int, copy=False))

    def minhash_many(self, X, device: int = 0) -> List[Optional[WeightedMinHash]]:
        """A matrix of weighted Jaccard vectors (rows; numpy or scipy.sparse) -> one WeightedMinHash per
        row, ``None`` for an all-zero row (weighted_minhash.py:161-247; same checks and return type).
        As there, the first negative or NaN weight of a row wins every sample, and a non-finite t (that one, or a
        +inf weight) is stored as INT64_MIN.

        The reference's experimental method rounds ``ln_a`` in a different order than ``minhash``
        (:221-224: ``ln_y = (t - beta + 1) * r; ln_a = ln_c - ln_y``); the kernel's
        ``DSK_WMH_MINHASH_MANY`` mode follows that order, so the values are the reference's
        ``minhash_many`` values, not necessarily ``minhash``'s.  A numpy matrix goes to the device in
        slabs of at most 256 MB; a scipy.sparse matrix goes as its stored entries (``dsk_wmh_minhash_csr``),
        with the same results as its densified rows."""
        sparse = hasattr(X, "tocsr") and hasattr(X, "nnz")
        if not sparse and not isinstance(X, np.ndarray):
            raise TypeError("Input X must be a sparse matrix or numpy matrix")
        if X.ndim != 2:
            raise ValueError("Input must have two dimensions")
        if X.shape[1] != self.dim:
            raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
        n = X.shape[0]
        ret: List[Optional[WeightedMinHash]] = [None] * n
        if sparse:
            out, status = self._sample_csr(X, device, many=True)
            for i in range(n):
                if status[i] != 1:
                    ret[i] = WeightedMinHash(self.seed, out[i].astype(int, copy=False))
            return ret
        slab = max(1, (256 << 20) // (4 * max(self.dim, 1)))
        for r0 in range(0, n, slab):
            part = X[r0:r0 + slab]
            dense = np.asarray(part, dtype=np.float32)
            out, status = self._sample(dense, device, many=True)
            for i in range(out.shape[0]):
                if status[i] != 1:
                    ret[r0 + i] = WeightedMinHash(self.seed, out[i].astype(int, copy=False))
        return ret
