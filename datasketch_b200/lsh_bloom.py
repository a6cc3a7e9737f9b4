"""MinHashLSHBloom -- the LSHBloom index (datasketch/lsh_bloom.py:125-380) with device-resident Bloom tables.

The reference keeps one Bloom filter per band and keys it with ``x = sum(band hashvalues) % (2**61 - 1)``
(``BloomTable.insert`` / ``query``, lsh_bloom.py:94-118); it can only answer "is this set a near-duplicate of
something inserted before?".  Same constructor, validation, ``BloomTable`` and ``insert`` / ``query`` / ``sync``
behaviour here; the bit tables live in HBM (``dsk_bloom_insert`` / ``dsk_bloom_query`` compute the band keys and
set / test the probe bits in one pass over the signature matrix) and ``insert_batch`` / ``query_batch`` take whole
matrices.  The reference delegates its bit tables to the optional ``pybloomfilter`` package; these tables are this
library's own classic k-probe Bloom filters sized by the same ``(item_count, fp)`` contract -- no false negatives,
false-positive rate <= fp at item_count insertions -- and ``*.bf`` files written by ``sync()`` hold this library's
format (a 32-byte header + the bit words), not pybloomfilter's mmap layout.
"""
from __future__ import annotations

import math
import os
import struct
import warnings
from typing import Optional, Tuple

import numpy as np

from . import _native as nv
from .lsh import _optimal_param, _signature_matrix

_mersenne_prime = np.uint64((1 << 61) - 1)
_MAGIC = b"DSKBLOOM"


def _bloom_size(item_count: int, fp: float) -> Tuple[int, int]:
    """Classic sizing: m = -n ln fp / (ln 2)^2 bits, k = (m / n) ln 2 probes."""
    n_bits = max(64, int(math.ceil(-item_count * math.log(fp) / (math.log(2.0) ** 2))))
    n_hashes = max(1, min(64, int(round(n_bits / item_count * math.log(2.0)))))
    return n_bits, n_hashes


class BloomTable:
    """One band's Bloom filter (datasketch/lsh_bloom.py:53-118): ``insert(hashvalues)`` / ``query(hashvalues)`` on the
    r hash values of a band, ``sync()`` to ``fname``.  The bits are a row of a CUDA tensor."""

    def __init__(self, item_count: int, fp: float, band_size: int, fname: Optional[str] = None, device: int = 0,
                 _bits=None):
        import torch
        self.r = band_size
        self.fname = fname
        self.device = device
        self.n_bits, self.n_hashes = _bloom_size(item_count, fp)
        self.words = (self.n_bits + 31) // 32
        nv.require_device(device)
        self.bits = _bits if _bits is not None else torch.zeros((self.words,), dtype=torch.int32,
                                                                device=torch.device("cuda", device))
        if fname is not None and os.path.exists(fname):
            with open(fname, "rb") as f:
                head = f.read(32)
                magic, n_bits, n_hashes, words = struct.unpack("<8sQQQ", head)
                if magic != _MAGIC or (n_bits, n_hashes, words) != (self.n_bits, self.n_hashes, self.words):
                    raise ValueError("%s does not hold a Bloom table for (item_count=%d, fp=%g)" % (fname, item_count, fp))
                saved = np.frombuffer(f.read(4 * words), dtype=np.uint32)
            self.bits.copy_(torch.from_numpy(saved.view(np.int32).copy()))

    def sync(self):
        if self.fname is None:
            warnings.warn("Attempting to save in-memory Bloom filter, this is a no-op.", RuntimeWarning, stacklevel=2)
            return
        with open(self.fname, "wb") as f:
            f.write(struct.pack("<8sQQQ", _MAGIC, self.n_bits, self.n_hashes, self.words))
            f.write(self.bits.cpu().numpy().view(np.uint32).tobytes())

    def assert_size(self, hashvalues):
        if not len(hashvalues) == self.r:
            raise RuntimeError(f"Invalid length for indices, {len(hashvalues)}, expected {self.r} hashvalues in band")

    def _row(self, hashvalues):
        import torch
        self.assert_size(hashvalues)
        hv = np.asarray(hashvalues)
        if hv.size and int(hv.max()) >= (1 << 32):
            raise ValueError("band hash values must fit 32 bits")
        return torch.from_numpy(np.ascontiguousarray(hv.astype(np.uint32)).view(np.int32).reshape(1, -1)).cuda(self.device)

    def insert(self, hashvalues) -> None:
        import torch
        row = self._row(hashvalues)   # one band of one signature = a [1, r] matrix with b = 1
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_bloom_insert(row.data_ptr(), 1, self.r, 1, self.r, self.bits.data_ptr(), self.words,
                                                self.n_bits, self.n_hashes, torch.cuda.current_stream().cuda_stream))

    def query(self, hashvalues) -> bool:
        import torch
        row = self._row(hashvalues)
        hit = torch.zeros((1,), dtype=torch.uint8, device=row.device)
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_bloom_query(row.data_ptr(), 1, self.r, 1, self.r, self.bits.data_ptr(), self.words,
                                               self.n_bits, self.n_hashes, hit.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
        return bool(hit.item())


def band_keys_host(hashvalues: np.ndarray, b: int, r: int) -> np.ndarray:
    """The b Bloom keys of ONE signature on the host, exactly as the reference computes them
    (``sum(hashvalues[start:end]) % _mersenne_prime``, lsh_bloom.py:105): API glue for single objects."""
    hv = np.asarray(hashvalues, dtype=np.uint64)
    return np.array([sum(hv[i * r:(i + 1) * r].tolist()) % int(_mersenne_prime) for i in range(b)], dtype=np.uint64)


class MinHashLSHBloom:
    """Drop-in for ``datasketch.MinHashLSHBloom`` (lsh_bloom.py:125): ``insert(minhash)``, ``query(minhash) -> bool``,
    ``sync()``, ``hashtables`` (one ``BloomTable`` per band); plus ``insert_batch(signatures)`` /
    ``query_batch(signatures) -> bool array`` on [N, K] matrices (one kernel launch each), and
    ``insert_unique(signatures) -> keep``, the query-then-insert de-duplication loop over a whole matrix."""

    def __init__(self, threshold: float = 0.9, num_perm: int = 128, n: Optional[int] = None, fp: Optional[float] = None,
                 save_dir: Optional[str] = None, weights: Tuple[float, float] = (0.5, 0.5),
                 params: Optional[Tuple[int, int]] = None, device: int = 0) -> None:
        # validation: the reference's, in its order (lsh_bloom.py:244-275)
        if threshold > 1.0 or threshold < 0.0:
            raise ValueError("threshold must be in [0.0, 1.0]")
        if num_perm < 2:
            raise ValueError("Too few permutation functions")
        if n is None or n <= 0:
            raise ValueError("n for LSHBloom must be >= 0")
        if fp is None or fp >= 1.0 or fp <= 0.0:
            raise ValueError("fp must be in (0.0, 1.0)")
        if save_dir is None:
            warnings.warn("Creating LSHBloom index without save directory, this index will not be persisted.",
                          RuntimeWarning, stacklevel=2)
        if any(w < 0.0 or w > 1.0 for w in weights):
            raise ValueError("Weight must be in [0.0, 1.0]")
        if sum(weights) != 1.0:
            raise ValueError("Weights must sum to 1.0")
        self.h = num_perm
        if params is not None:
            self.b, self.r = params
            if self.b * self.r > num_perm:
                raise ValueError(
                    "The product of b and r in params is "
                    f"{self.b} * {self.r} = {self.b * self.r} -- it must be less than num_perm {num_perm}. "
                    "Did you forget to specify num_perm?")
        else:
            self.b, self.r = _optimal_param(threshold, num_perm, weights[0], weights[1])
        if self.b < 2:
            raise ValueError("The number of bands are too small (b < 2)")
        import torch
        nv.require_device(device)
        self.device = device
        self.save_dir = save_dir
        self.n_bits, self.n_hashes = _bloom_size(n, fp)
        self.words_per_table = (self.n_bits + 31) // 32
        # one [b, words] tensor: the batch kernels address band j's table at row j; each BloomTable is a row view
        self._bits = torch.zeros((self.b, self.words_per_table), dtype=torch.int32, device=torch.device("cuda", device))
        if save_dir is not None:
            os.makedirs(save_dir, exist_ok=True)
        self.hashtables = [
            BloomTable(item_count=n, fp=fp, band_size=self.r,
                       fname=os.path.join(save_dir, f"band-{i}.bf") if save_dir is not None else None,
                       device=device, _bits=self._bits[i])
            for i in range(self.b)]
        self.hashranges = [(i * self.r, (i + 1) * self.r) for i in range(self.b)]

    # ---- whole matrices ---------------------------------------------------------------------------------------
    def _dev_sig(self, sig):
        import torch
        if isinstance(sig, np.ndarray):
            sig = torch.from_numpy(_signature_matrix(sig).view(np.int32)).cuda(self.device)
        if sig.dim() != 2 or sig.shape[1] != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, sig.shape[-1]))
        if sig.element_size() != 4:
            raise TypeError("MinHashLSHBloom takes the 32-bit signature matrix")
        return sig.contiguous()

    def insert_batch(self, signatures) -> None:
        """Insert every row of an [N, K] signature matrix (numpy uint32/uint64 or CUDA int32 tensor)."""
        import torch
        d_sig = self._dev_sig(signatures)
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_bloom_insert(d_sig.data_ptr(), d_sig.shape[0], self.h, self.b, self.r,
                                                self._bits.data_ptr(), self.words_per_table, self.n_bits, self.n_hashes,
                                                torch.cuda.current_stream().cuda_stream))

    def query_batch(self, signatures, to_host: bool = True):
        """bool per row: does ANY band of the row hit its Bloom table (lsh_bloom.py:365-371)?"""
        import torch
        d_sig = self._dev_sig(signatures)
        hit = torch.empty((d_sig.shape[0],), dtype=torch.uint8, device=d_sig.device)
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_bloom_query(d_sig.data_ptr(), d_sig.shape[0], self.h, self.b, self.r,
                                               self._bits.data_ptr(), self.words_per_table, self.n_bits, self.n_hashes,
                                               hit.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return hit.cpu().numpy().astype(bool) if to_host else hit.bool()

    def insert_unique(self, signatures, to_host: bool = True):
        """The streaming de-duplication loop over a whole [N, K] signature matrix, on the device::

            for m in rows:
                if not self.query(m):
                    self.insert(m)

        Returns ``keep``: ``keep[j]`` is True iff that loop, run over the rows in order from the tables as they are at
        the call, inserts row j.  The tables afterwards hold exactly the bits the loop leaves, i.e. their bits before
        the call plus ``insert_batch(signatures[keep])``.  Bloom false positives count exactly as the loop meets them:
        a band is covered when each of its probe bits is set, before the call or by kept rows earlier in the batch.
        ``query_batch`` followed by ``insert_batch`` of the misses is not the same: it keeps both rows of a
        near-duplicate pair inside one batch.

        Input as ``insert_batch``.  Stream-ordered with no host synchronisation (``to_host=False`` returns a CUDA bool
        tensor).  The workspace, about ``32 * b * n_hashes + 12`` bytes per row (``dsk_bloom_unique_workspace_size``),
        is allocated with torch; ``MemoryError`` names N and the bytes if it cannot be.  Batches of more than
        ``2^30 / (b * n_hashes)`` rows run as consecutive calls over slices, which give the same result."""
        import torch
        d_sig = self._dev_sig(signatures)
        n = d_sig.shape[0]
        keep = torch.empty((n,), dtype=torch.uint8, device=d_sig.device)
        lib = nv.load()
        step = max(1, (1 << 30) // (self.b * self.n_hashes))
        if n:
            need = int(lib.dsk_bloom_unique_workspace_size(min(n, step), self.h, self.b, self.r, self.n_hashes))
            try:
                ws = torch.empty((need,), dtype=torch.uint8, device=d_sig.device)
            except torch.OutOfMemoryError as exc:
                raise MemoryError("MinHashLSHBloom.insert_unique: cannot allocate the %d bytes of device memory the "
                                  "workspace needs for N = %d rows" % (need, min(n, step))) from exc
            with torch.cuda.device(self.device):
                stream = torch.cuda.current_stream().cuda_stream
                for lo in range(0, n, step):
                    rows = d_sig[lo:lo + step]
                    nv.check(lib.dsk_bloom_unique(rows.data_ptr(), rows.shape[0], self.h, self.b, self.r,
                                                  self._bits.data_ptr(), self.words_per_table, self.n_bits, self.n_hashes,
                                                  ws.data_ptr(), need, keep[lo:].data_ptr(), stream))
        return keep.cpu().numpy().astype(bool) if to_host else keep.bool()

    # ---- the reference's single-object API -------------------------------------------------------------------
    def _row(self, minhash) -> np.ndarray:
        if len(minhash) != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, len(minhash)))
        return np.asarray(minhash.hashvalues, dtype=np.uint64).reshape(1, -1)

    def insert(self, minhash) -> None:
        self.insert_batch(self._row(minhash))

    def _insert(self, minhash) -> None:
        self.insert(minhash)

    def query(self, minhash) -> bool:
        return bool(self.query_batch(self._row(minhash))[0])

    def sync(self) -> None:
        for table in self.hashtables:
            table.sync()
