"""Weighted MinHash with the reference's API (datasketch/weighted_minhash.py:11-159).

``WeightedMinHashGenerator.__init__`` draws the ICWS parameters on the host with numpy,
bit-identically to the reference (:118-121).  ``minhash`` (one vector) and
``minhash_batch`` (a matrix) run the per-sample argmin in ``libdsk_b200.so``
(``dsk_wmh_minhash``); every float32 step after ``log`` is IEEE-identical to numpy.
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
        ``GpuLSH(weighted=True)`` takes as it is: weights -> signatures -> index without a copy to the host."""
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
        ``minhash_many`` values, not necessarily ``minhash``'s.  Rows go to the device densified, in
        slabs of at most 256 MB."""
        sparse = hasattr(X, "tocsr") and hasattr(X, "nnz")
        if not sparse and not isinstance(X, np.ndarray):
            raise TypeError("Input X must be a sparse matrix or numpy matrix")
        if X.ndim != 2:
            raise ValueError("Input must have two dimensions")
        if X.shape[1] != self.dim:
            raise ValueError("Input dimension mismatch, expecting %d" % self.dim)
        if sparse:
            X = X.tocsr()
        n = X.shape[0]
        ret: List[Optional[WeightedMinHash]] = [None] * n
        slab = max(1, (256 << 20) // (4 * max(self.dim, 1)))
        for r0 in range(0, n, slab):
            part = X[r0:r0 + slab]
            dense = np.asarray(part.toarray() if sparse else part, dtype=np.float32)
            out, status = self._sample(dense, device, many=True)
            for i in range(out.shape[0]):
                if status[i] != 1:
                    ret[r0 + i] = WeightedMinHash(self.seed, out[i].astype(int, copy=False))
        return ret
