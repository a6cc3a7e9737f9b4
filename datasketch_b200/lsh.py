"""MinHashLSH with the reference's API (datasketch/lsh.py:51-668), plus batch / device paths.

Three layers:

* ``MinHashLSH`` -- the drop-in class over in-memory dict storage (the reference's default,
  storage.py:209-259): same constructor, ``insert / query / remove / merge / __contains__ /
  is_empty / get_counts / insertion_session ...``, same exceptions, same attributes
  (``b, r, h, hashranges, hashtables, keys``).  (b, r) come from the reference's optimiser
  (lsh.py:21-48; scipy ``quad`` on the host).  Redis / Cassandra / Mongo storage is network
  glue outside this engine's scope and raises ``ValueError``.
* ``MinHashLSH.insert_batch / query_batch`` -- the band keys ``_H`` builds one document at a
  time (lsh.py:344, :427, :537-538) are produced for a whole signature matrix by one kernel
  (``dsk_band_keys``) and then fed to the same dict buckets, so batch and per-item calls
  interoperate and produce the reference's bucket keys byte for byte.
* ``GpuLSH`` -- a device-resident index (``dsk_lsh_*``): insert and query never leave the GPU;
  candidate sets equal the reference's because buckets are verified on the r-tuples themselves.
"""
from __future__ import annotations

import ctypes
import pickle
import struct
from collections import defaultdict
from typing import Callable, Hashable, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np
from scipy.integrate import quad as integrate

from . import _native as nv
from . import codec
from .minhash import MinHash
from .weighted_minhash import WeightedMinHash


# ---- parameter optimiser (lsh.py:21-48): host-side, float64 -------------------------------------
def _false_positive_probability(threshold: float, b: int, r: int) -> float:
    area, _ = integrate(lambda s: 1 - (1 - s ** float(r)) ** float(b), 0.0, threshold)
    return area


def _false_negative_probability(threshold: float, b: int, r: int) -> float:
    area, _ = integrate(lambda s: 1 - (1 - (1 - s ** float(r)) ** float(b)), threshold, 1.0)
    return area


def _optimal_param(threshold: float, num_perm: int, false_positive_weight: float,
                   false_negative_weight: float) -> Tuple[int, int]:
    """Grid search over (b, r) with b*r <= num_perm; the first strict minimum wins."""
    best, opt = float("inf"), (0, 0)
    for b in range(1, num_perm + 1):
        for r in range(1, int(num_perm / b) + 1):
            err = (_false_positive_probability(threshold, b, r) * false_positive_weight
                   + _false_negative_probability(threshold, b, r) * false_negative_weight)
            if err < best:
                best, opt = err, (b, r)
    return opt


# ---- in-memory containers with the reference's Storage interface (storage.py:106-259) ------------
class _DictStorage:
    def __init__(self, factory):
        self._dict = defaultdict(factory)
        self._factory = factory

    def __getitem__(self, key):
        return self.get(key)

    def __delitem__(self, key):
        return self.remove(key)

    def __len__(self):
        return self.size()

    def __iter__(self):
        return iter(list(self._dict.keys()))

    def __contains__(self, item):
        return self.has_key(item)

    def keys(self):
        return self._dict.keys()

    def get(self, key):
        return self._dict.get(key, self._factory())

    def getmany(self, *keys):
        return [self.get(key) for key in keys]

    def remove(self, *keys, **kwargs):
        for key in keys:
            del self._dict[key]

    def size(self) -> int:
        return len(self._dict)

    def itemcounts(self, **kwargs) -> dict:
        return {k: len(v) for k, v in self._dict.items()}

    def has_key(self, key) -> bool:
        return key in self._dict

    def status(self):
        return {"keyspace_size": len(self)}

    # buffering is a no-op for in-memory storage
    buffer_size = 50000

    def empty_buffer(self):
        pass

    def add_to_select_buffer(self, keys):
        if not hasattr(self, "_select_buffer"):
            self._select_buffer = self.getmany(*keys)
        else:
            self._select_buffer.extend(self.getmany(*keys))

    def collect_select_buffer(self):
        if not hasattr(self, "_select_buffer"):
            return []
        buffered = list(self._select_buffer)
        del self._select_buffer[:]
        return buffered


class DictListStorage(_DictStorage):
    """key -> list of values (storage.py:209-244)."""

    def __init__(self, config=None):
        super().__init__(list)

    def remove_val(self, key, val, **kwargs):
        self._dict[key].remove(val)

    def insert(self, key, *vals, **kwargs):
        self._dict[key].extend(vals)


class DictSetStorage(_DictStorage):
    """key -> set of values (storage.py:247-259)."""

    def __init__(self, config=None):
        super().__init__(set)

    def remove_val(self, key, val, **kwargs):
        self._dict[key].remove(val)

    def insert(self, key, *vals, **kwargs):
        self._dict[key].update(vals)


def _storage(config: dict, ordered: bool):
    tp = config["type"]
    if tp == "dict":
        return DictListStorage(config) if ordered else DictSetStorage(config)
    raise ValueError("Unknown storage type: %s (this engine ships the in-memory 'dict' storage only)" % tp)


def _signature_matrix(minhashes) -> np.ndarray:
    """list of MinHash-like objects, or an [N, K] array -> contiguous uint32 [N, K]."""
    if isinstance(minhashes, np.ndarray):
        sig = minhashes
    else:
        sig = np.stack([np.asarray(m.hashvalues) for m in minhashes]) if len(minhashes) else np.zeros((0, 0), np.uint32)
    if sig.dtype != np.uint32:
        if sig.size and int(sig.max()) >= (1 << 32):
            raise ValueError("signature values must fit 32 bits")
        sig = sig.astype(np.uint32)
    return np.ascontiguousarray(sig)


class MinHashLSH:
    """The MinHash LSH index (constructor contract of lsh.py:147-200)."""

    def __init__(self, threshold: float = 0.9, num_perm: int = 128, weights: Tuple[float, float] = (0.5, 0.5),
                 params: Optional[Tuple[int, int]] = None, storage_config: Optional[dict] = None,
                 prepickle: Optional[bool] = None, hashfunc: Optional[Callable[[bytes], bytes]] = None) -> None:
        storage_config = storage_config if storage_config else {"type": "dict"}
        self._buffer_size = 50000
        if threshold > 1.0 or threshold < 0.0:
            raise ValueError("threshold must be in [0.0, 1.0]")
        if num_perm < 2:
            raise ValueError("Too few permutation functions")
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
            fpw, fnw = weights
            self.b, self.r = _optimal_param(threshold, num_perm, fpw, fnw)
        if self.b < 2:
            raise ValueError("The number of bands are too small (b < 2)")
        self.prepickle = storage_config["type"] == "redis" if prepickle is None else prepickle
        self._require_bytes_keys = not (storage_config["type"] == "dict" or self.prepickle)
        self.hashfunc = hashfunc
        self._H = self._hashed_byteswap if hashfunc else self._byteswap
        self.hashtables = [_storage(storage_config, ordered=False) for _ in range(self.b)]
        self.hashranges = [(i * self.r, (i + 1) * self.r) for i in range(self.b)]
        self.keys = _storage(storage_config, ordered=True)

    # -- buffer size plumbing (lsh.py:202-211) -------------------------------------------------------
    @property
    def buffer_size(self) -> int:
        return self._buffer_size

    @buffer_size.setter
    def buffer_size(self, value: int) -> None:
        self.keys.buffer_size = value
        for t in self.hashtables:
            t.buffer_size = value
        self._buffer_size = value

    # -- band keys --------------------------------------------------------------------------------------
    def _byteswap(self, hs) -> bytes:
        """One band's key: the r values as big-endian bytes (lsh.py:537-538)."""
        return bytes(np.asarray(hs).byteswap().data)

    def _hashed_byteswap(self, hs):
        if self.hashfunc is None:
            raise RuntimeError("Hash function not configured.")
        return self.hashfunc(self._byteswap(hs))

    def _batch_band_keys(self, sig: np.ndarray) -> List[List]:
        """GPU: all b band keys of every row of ``sig`` (uint32 [N, K]) -> per-row lists of keys."""
        if sig.shape[1] != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, sig.shape[1]))
        width = 8 * self.r
        raw = codec.band_keys(sig, self.b, self.r).cpu().numpy().reshape(len(sig), self.b * width).tobytes()
        row = self.b * width
        out = []
        for i in range(len(sig)):
            base = i * row
            ks = [raw[base + j * width: base + (j + 1) * width] for j in range(self.b)]
            out.append([self.hashfunc(k) for k in ks] if self.hashfunc else ks)
        return out

    # -- insert ---------------------------------------------------------------------------------------------
    def insert(self, key: Hashable, minhash: Union[MinHash, WeightedMinHash], check_duplication: bool = True):
        self._insert(key, minhash, check_duplication=check_duplication, buffer=False)

    def _check_key(self, key):
        if self._require_bytes_keys and not isinstance(key, bytes):
            raise TypeError(
                f"prepickle=False requires bytes keys for non-dict storage, got {type(key).__name__}. "
                "Either pass bytes keys or use prepickle=True for automatic serialization.")
        return pickle.dumps(key) if self.prepickle else key

    def _store(self, key, Hs, buffer: bool = False) -> None:
        self.keys.insert(key, *Hs, buffer=buffer)
        for H, hashtable in zip(Hs, self.hashtables):
            hashtable.insert(H, key, buffer=buffer)

    def _insert(self, key, minhash, check_duplication: bool = True, buffer: bool = False):
        if len(minhash) != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, len(minhash)))
        key = self._check_key(key)
        if check_duplication and key in self.keys:
            raise ValueError("The given key already exists")
        hv = minhash.hashvalues
        Hs = [self._H(hv[start:end]) for start, end in self.hashranges]
        self._store(key, Hs, buffer=buffer)

    def insert_batch(self, keys: Sequence[Hashable], minhashes, check_duplication: bool = True) -> None:
        """Insert many documents: one band-key kernel for the whole batch, then the bucket updates.

        ``minhashes`` is a list of MinHash / LeanMinHash objects or a uint32/uint64 [N, K] matrix."""
        sig = _signature_matrix(minhashes)
        if len(keys) != len(sig):
            raise ValueError("keys and minhashes differ in length")
        if len(sig) == 0:
            return
        skeys = [self._check_key(k) for k in keys]
        if check_duplication:
            seen = set()
            for k in skeys:
                if k in self.keys or k in seen:
                    raise ValueError("The given key already exists")
                seen.add(k)
        for k, Hs in zip(skeys, self._batch_band_keys(sig)):
            self._store(k, Hs)

    def export_redis(self, basename: bytes, prepickle: Optional[bool] = None):
        """This index in the reference's Redis layout (``storage_export.RedisLayout``; lsh.py:191-200,
        storage.py:902-1049): the state ``MinHashLSH(storage_config={"type": "redis", "basename": basename})`` would
        hold after the same inserts.  Keys are pickled unless ``prepickle=False`` (then they must be bytes)."""
        from .storage_export import RedisLayout
        prepickle = True if prepickle is None else prepickle
        layout = RedisLayout(basename, self.b)
        for key in self.keys.keys():
            hs = list(self.keys.get(key))
            stored = key
            if self.prepickle:                     # this index already holds pickled keys
                if not prepickle:
                    stored = pickle.loads(key)
            elif prepickle:
                stored = pickle.dumps(key)
            if not isinstance(stored, bytes):
                raise TypeError("prepickle=False requires bytes keys for non-dict storage, got %s" % type(stored).__name__)
            layout.add(stored, hs)
        return layout

    def export_cassandra(self, basename: bytes, prepickle: Optional[bool] = None):
        """This index in the reference's Cassandra layout (``storage_export.CassandraLayout``; lsh.py:191-200,
        storage.py:262-819): the rows ``MinHashLSH(storage_config={"type": "cassandra", "basename": basename, ...})`` would
        have written after the same inserts, in the same order.  ``prepickle`` defaults to False as for Cassandra in the
        reference (lsh.py:182): keys must then be bytes."""
        from .storage_export import CassandraLayout
        prepickle = False if prepickle is None else prepickle
        layout = CassandraLayout(basename, self.b)
        for key in self.keys.keys():
            hs = list(self.keys.get(key))
            stored = key
            if self.prepickle:                     # this index already holds pickled keys
                if not prepickle:
                    stored = pickle.loads(key)
            elif prepickle:
                stored = pickle.dumps(key)
            if not isinstance(stored, bytes):
                raise TypeError("prepickle=False requires bytes keys for non-dict storage, got %s" % type(stored).__name__)
            layout.add(stored, hs)
        return layout

    # -- merge (lsh.py:233-251, :349-368) -------------------------------------------------------------------------
    def merge(self, other: "MinHashLSH", check_overlap: bool = False):
        self._merge(other, check_overlap=check_overlap, buffer=False)

    def _equivalent(self, other) -> bool:
        return type(self) is type(other) and self.h == other.h and self.b == other.b and self.r == other.r

    def _merge(self, other, check_overlap: bool = False, buffer: bool = False) -> None:
        if self._equivalent(other):
            if check_overlap and set(self.keys).intersection(set(other.keys)):
                raise ValueError("The keys are overlapping, duplicate key exists.")
            for key in other.keys:
                self._store(key, other.keys.get(key), buffer=buffer)
        else:
            if type(self) is not type(other):
                raise ValueError(f"Cannot merge type MinHashLSH and type {type(other).__name__}.")
            raise ValueError("Cannot merge MinHashLSH with different initialization parameters.")

    # -- query ----------------------------------------------------------------------------------------------------------
    def query(self, minhash) -> list:
        """Keys whose sets likely exceed the Jaccard threshold (lsh.py:370-432)."""
        if len(minhash) != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, len(minhash)))
        candidates = set()
        hv = minhash.hashvalues
        for (start, end), hashtable in zip(self.hashranges, self.hashtables):
            for key in hashtable.get(self._H(hv[start:end])):
                candidates.add(key)
        if self.prepickle:
            return [pickle.loads(key) for key in candidates]
        return list(candidates)

    def query_batch(self, minhashes) -> List[list]:
        """``[self.query(m) for m in minhashes]`` with the band keys of all queries built by one kernel."""
        sig = _signature_matrix(minhashes)
        if len(sig) == 0:
            return []
        out = []
        for Hs in self._batch_band_keys(sig):
            cand = set()
            for H, hashtable in zip(Hs, self.hashtables):
                cand.update(hashtable.get(H))
            out.append([pickle.loads(k) for k in cand] if self.prepickle else list(cand))
        return out

    def add_to_query_buffer(self, minhash) -> None:
        if len(minhash) != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, len(minhash)))
        hv = minhash.hashvalues
        for (start, end), hashtable in zip(self.hashranges, self.hashtables):
            hashtable.add_to_select_buffer([self._H(hv[start:end])])

    def collect_query_buffer(self) -> list:
        """Intersection over buffered queries of the per-query unions over bands (lsh.py:455-484)."""
        collected = [hashtable.collect_select_buffer() for hashtable in self.hashtables]
        if not any(collected):
            return []
        per_query = [set().union(*lists) for lists in zip(*collected)]
        if not per_query:
            return []
        candidates = set.intersection(*per_query)
        if self.prepickle:
            return [pickle.loads(key) for key in candidates]
        return list(candidates)

    # -- membership / removal -------------------------------------------------------------------------------------------------
    def __contains__(self, key: Hashable) -> bool:
        if self.prepickle:
            key = pickle.dumps(key)
        return key in self.keys

    def remove(self, key: Hashable) -> None:
        self._remove(key, buffer=False)

    def _remove(self, key: Hashable, buffer: bool = False) -> None:
        if self.prepickle:
            key = pickle.dumps(key)
        if key not in self.keys:
            raise ValueError("The given key does not exist")
        for H, hashtable in zip(self.keys[key], self.hashtables):
            hashtable.remove_val(H, key, buffer=buffer)
            if not hashtable.get(H):
                hashtable.remove(H, buffer=buffer)
        self.keys.remove(key, buffer=buffer)

    def is_empty(self) -> bool:
        return any(t.size() == 0 for t in self.hashtables)

    def _query_b(self, minhash, b: int):
        if len(minhash) != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, len(minhash)))
        if b > len(self.hashtables):
            raise ValueError("b must be less or equal to the number of hash tables")
        candidates = set()
        hv = minhash.hashvalues
        for (start, end), hashtable in zip(self.hashranges[:b], self.hashtables[:b]):
            H = self._H(hv[start:end])
            if H in hashtable:
                for key in hashtable[H]:
                    candidates.add(key)
        if self.prepickle:
            return {pickle.loads(key) for key in candidates}
        return candidates

    def get_counts(self) -> List[dict]:
        return [hashtable.itemcounts() for hashtable in self.hashtables]

    def get_subset_counts(self, *keys: Hashable) -> List[dict]:
        key_set = [pickle.dumps(key) for key in set(keys)] if self.prepickle else list(set(keys))
        tables = [DictSetStorage() for _ in range(self.b)]
        for key, Hs in zip(key_set, self.keys.getmany(*key_set)):
            for H, table in zip(Hs, tables):
                table.insert(H, key)
        return [table.itemcounts() for table in tables]

    # -- sessions (lsh.py:253-324, :592-668) -----------------------------------------------------------------------------------
    def insertion_session(self, buffer_size: int = 50000) -> "MinHashLSHInsertionSession":
        return MinHashLSHInsertionSession(self, buffer_size=buffer_size)

    def deletion_session(self, buffer_size: int = 50000) -> "MinHashLSHDeletionSession":
        return MinHashLSHDeletionSession(self, buffer_size=buffer_size)


class MinHashLSHInsertionSession:
    """Context manager for batch insertion (lsh.py:592-634)."""

    def __init__(self, lsh: MinHashLSH, buffer_size: int):
        self.lsh = lsh
        self.lsh.buffer_size = buffer_size

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_val, exc_tb) -> None:
        self.close()

    def close(self) -> None:
        self.lsh.keys.empty_buffer()
        for hashtable in self.lsh.hashtables:
            hashtable.empty_buffer()

    def insert(self, key, minhash, check_duplication: bool = True) -> None:
        self.lsh._insert(key, minhash, check_duplication=check_duplication, buffer=True)


class MinHashLSHDeletionSession:
    """Context manager for batch deletion (lsh.py:637-668)."""

    def __init__(self, lsh: MinHashLSH, buffer_size: int):
        self.lsh = lsh
        self.lsh.buffer_size = buffer_size

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_val, exc_tb) -> None:
        self.close()

    def close(self) -> None:
        self.lsh.keys.empty_buffer()
        for hashtable in self.lsh.hashtables:
            hashtable.empty_buffer()

    def remove(self, key) -> None:
        self.lsh._remove(key, buffer=True)


# ---- device-resident index -----------------------------------------------------------------------------
class GpuLSH:
    """Device-resident MinHashLSH buckets: ``insert`` / ``query`` over whole signature matrices.

    Same banding as ``MinHashLSH`` (pass ``threshold``/``weights`` or ``params``); documents are
    numbered in insertion order and ``keys`` (optional) maps numbers to user keys.  ``query``
    returns CSR arrays ``(ptr, idx)``: the candidates of query ``q`` are ``idx[ptr[q]:ptr[q+1]]``
    -- as a set, exactly ``MinHashLSH.query`` on the same data.

    ``weighted=True`` indexes weighted MinHash signatures, as ``MinHashLSH(num_perm=ss)`` does with
    ``WeightedMinHash`` objects: ``num_perm`` is the sample size ss, ``(b, r)`` count samples, and every method
    that takes signatures takes ``[N, ss, 2]`` integer ``(k, t)`` rows (a numpy array, a CUDA tensor as
    ``WeightedMinHashGenerator.minhash_batch(..., to_host=False)`` returns it, or a list of ``WeightedMinHash``)
    with ``0 <= k < 2^32`` and ``-2^31 <= t < 2^31``.  Every ``eq`` then counts the samples whose ``(k, t)``
    pairs agree, so ``eq / num_perm`` is ``WeightedMinHash.jaccard``, and the candidate sets are the reference's.
    """

    def __init__(self, threshold: float = 0.9, num_perm: int = 128, weights: Tuple[float, float] = (0.5, 0.5),
                 params: Optional[Tuple[int, int]] = None, capacity: int = 1 << 20, device: int = 0,
                 weighted: bool = False):
        if params is not None:
            self.b, self.r = params
            if self.b * self.r > num_perm:
                raise ValueError("The product of b and r in params must be less than num_perm")
        else:
            if threshold > 1.0 or threshold < 0.0:
                raise ValueError("threshold must be in [0.0, 1.0]")
            self.b, self.r = _optimal_param(threshold, num_perm, weights[0], weights[1])
        if self.b < 2:
            raise ValueError("The number of bands are too small (b < 2)")
        self.h = num_perm
        self.weighted = bool(weighted)
        self.device = device
        self.capacity = int(capacity)
        nv.require_device(device)
        h = ctypes.c_void_p()
        create = nv.load().dsk_lsh_create_weighted if self.weighted else nv.load().dsk_lsh_create
        nv.check(create(num_perm, self.b, self.r, self.capacity, device, ctypes.byref(h)))
        self._h = h
        self.keys: List[Hashable] = []

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                nv.load().dsk_lsh_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass

    def __len__(self) -> int:
        n = ctypes.c_int64()
        nv.check(nv.load().dsk_lsh_size(self._h, ctypes.byref(n), None))
        return int(n.value)

    def _dev_sig(self, sig):
        import torch
        if self.weighted:
            return _pack_weighted(sig, self.h, torch.device("cuda", self.device))
        if isinstance(sig, np.ndarray):
            sig = torch.from_numpy(_signature_matrix(sig).view(np.int32)).cuda(self.device)
        if sig.dim() != 2 or sig.shape[1] != self.h:
            raise ValueError("Expecting minhash with length %d, got %d" % (self.h, sig.shape[-1]))
        if sig.element_size() != 4:
            raise TypeError("GpuLSH takes the 32-bit signature matrix")
        return sig.contiguous()

    def insert(self, sig, keys: Optional[Iterable[Hashable]] = None) -> None:
        """Append the rows of ``sig`` ([N, K] uint32; numpy or CUDA tensor) to the index."""
        import torch
        d_sig = self._dev_sig(sig)
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_lsh_insert(self._h, d_sig.data_ptr(), d_sig.shape[0],
                                              torch.cuda.current_stream().cuda_stream))
        if keys is not None:
            self.keys.extend(keys)

    def insert_tokens(self, d_tokens, d_offsets, n_tokens: int, permutations: np.ndarray,
                      keys: Optional[Iterable[Hashable]] = None) -> None:
        """Append documents given as TOKEN lists (CUDA tensors: uint32/int32 or uint64/int64 hash values, int64 CSR
        offsets): ``MinHash.bulk`` + ``insert`` of every document (minhash.py:464-489, lsh.py:326-347) in one launch --
        the signature kernel builds each row straight into the index's storage and the warp that finishes a row does
        its bucket updates (``dsk_lsh_insert_tokens``).  ``permutations`` is the (2, K) array of ``MinHash.permutations``.
        Not available on a weighted index (tokens give MinHash rows)."""
        import torch
        if self.weighted:
            raise ValueError("insert_tokens builds MinHash rows; a weighted index takes weighted MinHash signatures")
        if not d_tokens.is_cuda or not d_offsets.is_cuda or d_tokens.device.index != self.device \
                or d_offsets.device.index != self.device:
            raise ValueError("insert_tokens needs CUDA tensors on device %d" % self.device)
        if d_offsets.dtype != torch.int64 or d_offsets.dim() != 1 or d_offsets.numel() < 1 or not d_offsets.is_contiguous():
            raise ValueError("offsets must be a contiguous 1-D int64 tensor of length n_docs + 1")
        if d_tokens.element_size() not in (4, 8) or d_tokens.is_floating_point() or not d_tokens.is_contiguous():
            raise ValueError("tokens must be a contiguous 32-bit or 64-bit integer tensor")
        if int(n_tokens) > d_tokens.numel():
            raise ValueError("n_tokens exceeds the token tensor")
        hp = nv.perm_handle(permutations, self.device)
        if hp.num_perm != self.h:
            raise ValueError("Expecting permutations of length %d, got %d" % (self.h, hp.num_perm))
        n = d_offsets.numel() - 1
        with torch.cuda.device(self.device):
            nv.check(nv.load().dsk_lsh_insert_tokens(self._h, hp.handle, d_tokens.data_ptr() if n_tokens else None,
                                                     int(d_tokens.element_size() == 8), d_offsets.data_ptr(), n, int(n_tokens),
                                                     torch.cuda.current_stream().cuda_stream))
        if keys is not None:
            self.keys.extend(keys)

    def query(self, sig, to_host: bool = True):
        """Candidates of every row of ``sig``: ``(ptr int64[Q+1], idx int32[total])``."""
        import torch
        d_q = self._dev_sig(sig)
        nq = d_q.shape[0]
        dev = d_q.device
        lib = nv.load()
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            counts = torch.empty((max(nq, 1),), dtype=torch.int64, device=dev)
            ptr = torch.empty((nq + 1,), dtype=torch.int64, device=dev)
            scratch = torch.empty((nq // 1024 + 2,), dtype=torch.int64, device=dev)
            nv.check(lib.dsk_lsh_query_count(self._h, d_q.data_ptr(), nq, counts.data_ptr(), st))
            nv.check(lib.dsk_exclusive_scan(counts.data_ptr(), nq, ptr.data_ptr(), scratch.data_ptr(), st))
            total = int(ptr[nq].item())
            idx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            nv.check(lib.dsk_lsh_query_fill(self._h, d_q.data_ptr(), nq, ptr.data_ptr(), idx.data_ptr(), st))
            idx = idx[:total]
        if to_host:
            return ptr.cpu().numpy(), idx.cpu().numpy()
        return ptr, idx

    def query_keys(self, sig) -> List[list]:
        """Like ``MinHashLSH.query_batch``: per query, the list of user keys (or document numbers)."""
        ptr, idx = self.query(sig)
        out = []
        for q in range(len(ptr) - 1):
            ids = idx[ptr[q]:ptr[q + 1]]
            out.append([self.keys[i] for i in ids] if self.keys else ids.tolist())
        return out

    # -- queries verified on the device: Jaccard counts, a min_jaccard filter and each query's best match -------------
    def query_jaccard(self, sig, min_jaccard: Optional[float] = None, to_host: bool = True):
        """Candidates of every row of ``sig`` with their Jaccard counts: ``(ptr int64[Q+1], idx int32[M], eq int32[M])``.

        ``idx[ptr[q]:ptr[q+1]]`` lists each candidate of query q once, in no particular order; without ``min_jaccard``
        the candidates, as a set, are ``query(sig)``'s.  ``eq`` is the number of the ``num_perm`` positions where the query
        row and the document's row agree, so ``eq / num_perm`` is ``MinHash.jaccard`` (on a weighted index: the samples
        whose ``(k, t)`` pairs agree, and ``WeightedMinHash.jaccard``).  ``min_jaccard`` keeps only the
        candidates with ``MinHash.jaccard >= min_jaccard``: ``[d for d in lsh.query(m) if m.jaccard(doc[d]) >= t]`` for
        every query at once, on the rows the index holds.  A query costs time linear in the size of the buckets it hits."""
        import torch
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_q = self._dev_sig(sig)
        nq = d_q.shape[0]
        dev = d_q.device
        lib = nv.load()
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            counts = torch.empty((max(nq, 1),), dtype=torch.int64, device=dev)
            ptr = torch.empty((nq + 1,), dtype=torch.int64, device=dev)
            scratch = torch.empty((nq // 1024 + 2,), dtype=torch.int64, device=dev)
            nv.check(lib.dsk_lsh_query_jaccard_count(self._h, d_q.data_ptr(), nq, mc, counts.data_ptr(), st))
            nv.check(lib.dsk_exclusive_scan(counts.data_ptr(), nq, ptr.data_ptr(), scratch.data_ptr(), st))
            total = int(ptr[nq].item())
            idx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            eq = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            nv.check(lib.dsk_lsh_query_jaccard_fill(self._h, d_q.data_ptr(), nq, mc, ptr.data_ptr(), idx.data_ptr(),
                                                    eq.data_ptr(), st))
            idx, eq = idx[:total], eq[:total]
        if to_host:
            return ptr.cpu().numpy(), idx.cpu().numpy(), eq.cpu().numpy()
        return ptr, idx, eq

    def query_best(self, sig, min_jaccard: Optional[float] = None, to_host: bool = True):
        """Each query's closest indexed document: ``(idx int32[Q], eq int32[Q])``, the candidate of ``query_jaccard(sig,
        min_jaccard)`` with the largest ``eq``, the smallest document number among equal ones.  Both are -1 where the
        query keeps no candidate.  ``eq / num_perm`` is the query's largest ``MinHash.jaccard`` over its candidates, e.g. a
        document's similarity to the corpus in a decontamination report.  One launch, without a host synchronisation."""
        import torch
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_q = self._dev_sig(sig)
        nq = d_q.shape[0]
        with torch.cuda.device(self.device):
            idx = torch.empty((max(nq, 1),), dtype=torch.int32, device=d_q.device)
            eq = torch.empty((max(nq, 1),), dtype=torch.int32, device=d_q.device)
            nv.check(nv.load().dsk_lsh_query_best(self._h, d_q.data_ptr(), nq, mc, idx.data_ptr(), eq.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream))
            idx, eq = idx[:nq], eq[:nq]
        if to_host:
            return idx.cpu().numpy(), eq.cpu().numpy()
        return idx, eq

    # -- the k most similar candidates, ranked on the device ---------------------------------------------------------------
    def query_topk(self, sig, k: int, min_jaccard: Optional[float] = None, to_host: bool = True):
        """Each query's k most similar indexed documents: ``(idx int32[Q, k], eq int32[Q, k])``.

        Row q holds the first k candidates of ``query_jaccard(sig, min_jaccard)`` for query q in the order larger ``eq``
        first, then smaller document number (a total order, so the result is fixed), best first; the slots behind them
        are -1 / -1.  ``eq / num_perm`` is ``MinHash.jaccard`` (``WeightedMinHash.jaccard`` on a weighted index).  For a
        query m this is::

            sorted([d for d in lsh.query(m) if m.jaccard(doc[d]) >= t], key=lambda d: (-m.jaccard(doc[d]), d))[:k]

        ``k`` is in ``[1, 32]``; ``query_topk(sig, 1)`` equals ``query_best(sig)``.  Removed documents are never listed.
        One launch, without a host synchronisation, and an output of ``Q * k`` entries however many candidates a query
        has; the walk and the verification cost what ``query_jaccard``'s do."""
        import torch
        k = _check_topk(k)
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_q = self._dev_sig(sig)
        nq = d_q.shape[0]
        with torch.cuda.device(self.device):
            idx = torch.empty((max(nq, 1), k), dtype=torch.int32, device=d_q.device)
            eq = torch.empty((max(nq, 1), k), dtype=torch.int32, device=d_q.device)
            nv.check(nv.load().dsk_lsh_query_topk(self._h, d_q.data_ptr(), nq, mc, k, idx.data_ptr(), eq.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream))
            idx, eq = idx[:nq], eq[:nq]
        if to_host:
            return idx.cpu().numpy(), eq.cpu().numpy()
        return idx, eq

    def neighbors(self, k: int, min_jaccard: Optional[float] = None, to_host: bool = True):
        """The k nearest neighbours of every indexed document: ``(idx int32[n, k], eq int32[n, k])``, ``n = len(self)``.

        Row i is ``query_topk``'s list for document i's own row with i itself left out: every other document d, below
        or above i, that ``query`` returns for row i and that ``min_jaccard`` keeps, in the order larger ``eq`` first,
        then smaller d, cut at k; -1 / -1 behind them.  For document i with row m this is::

            sorted([d for d in lsh.query(m) if d != i and m.jaccard(doc[d]) >= t],
                   key=lambda d: (-m.jaccard(doc[d]), d))[:k]

        ``k`` is in ``[1, 32]``.  A removed document's row is all -1 and it appears in no list; after ``compact()`` rows
        and numbers follow its ``remap``.  One launch, without a host synchronisation.  Each pair is verified from both
        ends, about twice the row comparisons of ``candidate_pairs``: still quadratic in the size of each bucket; only
        the output is bounded."""
        import torch
        k = _check_topk(k)
        mc = _jaccard_min_count(min_jaccard, self.h)
        n = len(self)
        with torch.cuda.device(self.device):
            dev = torch.device("cuda", self.device)
            idx = torch.empty((max(n, 1), k), dtype=torch.int32, device=dev)
            eq = torch.empty((max(n, 1), k), dtype=torch.int32, device=dev)
            nv.check(nv.load().dsk_lsh_neighbors(self._h, mc, k, idx.data_ptr(), eq.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream))
            idx, eq = idx[:n], eq[:n]
        if to_host:
            return idx.cpu().numpy(), eq.cpu().numpy()
        return idx, eq

    # -- streaming de-duplication: insert the rows that have no near-duplicate yet ---------------------------------------
    def insert_unique(self, sig, min_jaccard: Optional[float] = None, keys: Optional[Iterable[Hashable]] = None,
                      to_host: bool = True):
        """Insert the rows of ``sig`` that have no near-duplicate yet: ``(kept bool[B], match int32[B], eq int32[B])``.

        The result is, row for row, that of the streaming de-duplication loop over the batch in order::

            for j, m in enumerate(sig):
                if not [d for d in lsh.query(m) if m.jaccard(doc[d]) >= min_jaccard]:
                    lsh.insert(key[j], m)

        Row j is kept iff no remaining (not removed) document of the index and no row of this batch kept before j is a
        candidate of row j with ``MinHash.jaccard >= min_jaccard`` (``min_jaccard=None``: any candidate drops the row).
        The kept rows become documents ``len(self), len(self) + 1, ...`` in batch order, and ``keys`` (one per row, when
        given) is appended for the kept rows only.  For a dropped row, ``match`` / ``eq`` give the candidate of the loop's
        query with the largest ``eq`` (the number of agreeing positions; ``eq / num_perm`` is ``MinHash.jaccard``), the
        smallest document number among equal ones, with the numbers the documents have after the call: an indexed
        document wins a tie against a row of the batch.  Both are -1 for a kept row.

        This differs from ``duplicate_clusters``, which keeps one document per connected component: in a drift chain
        a ~ b ~ c where a and c do not match, the loop keeps a and c (b is dropped, so nothing kept matches c), while
        the component {a, b, c} keeps only a.

        If the kept rows do not fit the capacity, raises ``ValueError`` and changes nothing: the index, ``len()`` and
        ``keys`` are as before.  Runs on the device and waits for it twice: for the size of the batch's pair list and
        for the number of kept rows."""
        import torch
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_sig = self._dev_sig(sig)
        n = d_sig.shape[0]
        if keys is not None:
            keys = list(keys)
            if len(keys) != n:
                raise ValueError("keys must hold one key per row of sig (%d), got %d" % (n, len(keys)))
        lib = nv.load()
        dev = d_sig.device
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            ws_bytes = int(lib.dsk_lsh_unique_workspace_size(self._h, n))
            ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
            counts = torch.empty((max(n, 1),), dtype=torch.int64, device=dev)
            ptr = torch.empty((n + 1,), dtype=torch.int64, device=dev)
            scratch = torch.empty((n // 1024 + 2,), dtype=torch.int64, device=dev)
            nv.check(lib.dsk_lsh_unique_count(self._h, d_sig.data_ptr(), n, mc, ws.data_ptr(), ws_bytes,
                                              counts.data_ptr(), st))
            nv.check(lib.dsk_exclusive_scan(counts.data_ptr(), n, ptr.data_ptr(), scratch.data_ptr(), st))
            total = int(ptr[n].item())
            pidx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            peq = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            kept = torch.empty((max(n, 1),), dtype=torch.uint8, device=dev)
            match = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
            eq = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
            inserted = ctypes.c_int64(0)
            nv.check(lib.dsk_lsh_unique_commit(self._h, d_sig.data_ptr(), n, mc, ws.data_ptr(), ws_bytes, ptr.data_ptr(),
                                               pidx.data_ptr(), peq.data_ptr(), kept.data_ptr(), match.data_ptr(),
                                               eq.data_ptr(), ctypes.byref(inserted), st))
            kept, match, eq = kept[:n].bool(), match[:n], eq[:n]
        if keys is not None:
            mask = kept.cpu().numpy()
            self.keys.extend(k for k, keep in zip(keys, mask) if keep)
        if to_host:
            return kept.cpu().numpy(), match.cpu().numpy(), eq.cpu().numpy()
        return kept, match, eq

    # -- self-join: near-duplicate pairs and clusters of the indexed documents ------------------------------------------
    def candidate_pairs(self, min_jaccard: Optional[float] = None, to_host: bool = True):
        """Every candidate pair among the ``n = len(self)`` indexed documents, once, as CSR arrays
        ``(ptr int64[n+1], idx int32[M], eq int32[M])``.

        ``idx[ptr[i]:ptr[i+1]]`` holds (unordered) the documents ``d < i`` that ``query`` returns for document i's own row,
        and ``eq`` the number of the ``num_perm`` positions where the two rows agree, so ``eq / num_perm`` is
        ``MinHash.jaccard`` of the pair (``WeightedMinHash.jaccard`` on a weighted index, where eq counts samples).
        ``min_jaccard`` keeps only the pairs with ``MinHash.jaccard >= min_jaccard``.
        Runs on the device: one warp per document walks the document's buckets and compares the rows the index holds."""
        import torch
        mc = _jaccard_min_count(min_jaccard, self.h)
        n = len(self)
        lib = nv.load()
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            counts = torch.empty((max(n, 1),), dtype=torch.int64, device=dev)
            ptr = torch.empty((n + 1,), dtype=torch.int64, device=dev)
            scratch = torch.empty((n // 1024 + 2,), dtype=torch.int64, device=dev)
            nv.check(lib.dsk_lsh_pairs_count(self._h, mc, counts.data_ptr(), st))
            nv.check(lib.dsk_exclusive_scan(counts.data_ptr(), n, ptr.data_ptr(), scratch.data_ptr(), st))
            total = int(ptr[n].item())
            idx = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            eq = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
            nv.check(lib.dsk_lsh_pairs_fill(self._h, mc, ptr.data_ptr(), idx.data_ptr(), eq.data_ptr(), st))
            idx, eq = idx[:total], eq[:total]
        if to_host:
            return ptr.cpu().numpy(), idx.cpu().numpy(), eq.cpu().numpy()
        return ptr, idx, eq

    def duplicate_clusters(self, min_jaccard: Optional[float] = None, to_host: bool = True):
        """``labels int32[n]``: ``labels[i]`` is the smallest document number of i's connected component in the graph of
        ``candidate_pairs(min_jaccard)``.  Deterministic; ``labels[i] == i`` marks the one document of each cluster a
        de-duplication keeps, and ``keys`` (when set) maps labels to user keys.

        Without ``min_jaccard`` each document is linked to the first equal member of each of its buckets, which takes
        time linear in the index however large its buckets are.  With ``min_jaccard`` every candidate pair is verified,
        which takes time quadratic in the size of each bucket."""
        import torch
        mc = _jaccard_min_count(min_jaccard, self.h)
        n = len(self)
        with torch.cuda.device(self.device):
            labels = torch.empty((max(n, 1),), dtype=torch.int32, device=torch.device("cuda", self.device))
            nv.check(nv.load().dsk_lsh_clusters(self._h, mc, labels.data_ptr(), torch.cuda.current_stream().cuda_stream))
            labels = labels[:n]
        return labels.cpu().numpy() if to_host else labels

    # -- removal and compaction (MinHashLSH.remove, lsh.py:497-528) ----------------------------------------------------
    def _doc_tensor(self, docs):
        """``docs`` (one number, a sequence, a numpy array or a CUDA tensor) as a 1-D int64 CUDA tensor."""
        import torch
        dev = torch.device("cuda", self.device)
        if isinstance(docs, torch.Tensor):
            if docs.is_floating_point() or docs.is_complex() or docs.dtype == torch.bool:
                raise TypeError("document numbers must be integers")
            return docs.reshape(-1).to(device=dev, dtype=torch.int64)
        a = np.asarray(docs).reshape(-1)
        if a.size and a.dtype.kind not in "iu":
            raise TypeError("document numbers must be integers")
        return torch.from_numpy(a.astype(np.int64)).to(dev)

    def remove(self, docs) -> None:
        """Remove documents (their numbers: one, a sequence, a numpy array or a CUDA tensor) from the index, as
        ``MinHashLSH.remove`` removes keys.  Afterwards ``query`` never returns them, ``candidate_pairs`` pairs nothing
        with them (their own rows are empty) and ``duplicate_clusters`` labels them -1; the pairs and clusters of the
        remaining documents are those before the removal restricted to them.

        Document numbers do not change until ``compact()``, and ``len()`` still counts removed documents until then.
        Raises ``ValueError("The given key does not exist")`` if a number is out of range, already removed or listed twice;
        the index is then unchanged (everything is checked before anything is removed)."""
        import torch
        d = self._doc_tensor(docs)
        n = len(self)
        if d.numel() == 0:
            return
        if bool(((d < 0) | (d >= n)).any()) or torch.unique(d).numel() != d.numel():
            raise ValueError("The given key does not exist")
        d32 = d.to(torch.int32)
        if not bool(self._alive(d32).all()):
            raise ValueError("The given key does not exist")
        with torch.cuda.device(self.device):
            status = torch.zeros((2,), dtype=torch.int64, device=d32.device)
            nv.check(nv.load().dsk_lsh_remove(self._h, d32.data_ptr(), d32.numel(), status.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))

    def _alive(self, d32):
        import torch
        with torch.cuda.device(self.device):
            out = torch.empty((max(d32.numel(), 1),), dtype=torch.uint8, device=d32.device)
            nv.check(nv.load().dsk_lsh_alive(self._h, d32.data_ptr(), d32.numel(), out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
        return out[:d32.numel()].bool()

    def alive(self, docs=None, to_host: bool = True):
        """Bool mask: True where the document number is in ``[0, len(self))`` and not removed.  Over ``docs``, or over all
        ``len(self)`` numbers when ``docs`` is None."""
        import torch
        if docs is None:
            d32 = torch.arange(len(self), dtype=torch.int32, device=torch.device("cuda", self.device))
        else:
            d = self._doc_tensor(docs)
            d32 = torch.where((d >= 0) & (d < (1 << 31)), d, torch.full_like(d, -1)).to(torch.int32)
        mask = self._alive(d32)
        return mask.cpu().numpy() if to_host else mask

    def compact(self, to_host: bool = True):
        """Renumber the remaining documents ``0..m-1`` in their old order, rebuild the buckets from them and free the
        capacity the removed ones held.  Returns ``remap`` (int32, one entry per old number: the new number, or -1 for a
        removed document).  Because the order is kept, ``candidate_pairs`` afterwards equals the earlier pairs mapped
        through ``remap``, ``duplicate_clusters`` equals ``remap[labels_before]`` on the remaining documents, and the
        index behaves as a fresh ``GpuLSH`` into which the remaining rows were inserted in order.  ``keys``, when it
        holds one key per document, keeps the remaining keys.  Waits for the device once."""
        import torch
        n = len(self)
        lib = nv.load()
        dev = torch.device("cuda", self.device)
        with torch.cuda.device(self.device):
            ws_bytes = int(lib.dsk_lsh_compact_workspace_size(self._h))
            ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
            remap = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
            nv.check(lib.dsk_lsh_compact(self._h, remap.data_ptr(), ws.data_ptr(), ws_bytes,
                                         torch.cuda.current_stream().cuda_stream))
            remap = remap[:n]
        if self.keys and len(self.keys) == n:
            keep = remap.cpu().numpy() >= 0
            self.keys = [k for k, kept in zip(self.keys, keep) if kept]
        return remap.cpu().numpy() if to_host else remap


_WMH_K_MAX = (1 << 32) - 1                      # k is packed as uint32
_WMH_T_MIN, _WMH_T_MAX = -(1 << 31), (1 << 31) - 1   # t is packed as int32


def _pack_weighted(sig, sample_size: int, device):
    """Weighted MinHash rows -> the ``[N, 2 * sample_size]`` int32 tensor a weighted ``GpuLSH`` holds, on ``device``
    (anything ``torch.device`` takes; the index passes its CUDA device).

    ``sig`` is an ``[N, sample_size, 2]`` integer array of ``(k, t)`` pairs (numpy or a CUDA tensor) or a list of
    ``WeightedMinHash``.  Sample j becomes word 2j = k_j as uint32 and word 2j + 1 = t_j as int32 (two's complement).  On
    ``0 <= k < 2^32``, ``-2^31 <= t < 2^31`` the packing is injective, so equal words are equal pairs; values outside
    raise ``ValueError`` naming the bound, before anything is sent to the index."""
    import torch
    dev = torch.device(device)
    if isinstance(sig, torch.Tensor):
        if sig.is_floating_point() or sig.is_complex() or sig.dtype in (torch.bool, torch.uint64):
            raise TypeError("weighted MinHash rows must be a signed (or 8/16/32-bit unsigned) integer tensor")
        x = sig.to(device=dev, dtype=torch.int64)   # exact for these types; the range is then checked on the device
    else:
        if not isinstance(sig, np.ndarray):
            sig = list(sig)
            sig = np.stack([np.asarray(m.hashvalues) for m in sig]) if sig else np.zeros((0, sample_size, 2), np.int64)
        if sig.dtype.kind not in "iu":
            raise TypeError("weighted MinHash rows must be integers")
        x = sig
    if x.ndim != 3 or x.shape[1] != sample_size or x.shape[2] != 2:
        raise ValueError("Expecting weighted minhash rows of shape [N, %d, 2], got %s" % (sample_size, tuple(x.shape)))
    k, t = x[..., 0], x[..., 1]
    if x.shape[0]:
        if bool((k < 0).any()) or bool((k > _WMH_K_MAX).any()):
            raise ValueError("weighted MinHash k values must be in [0, 2^32 - 1]")
        if bool((t < _WMH_T_MIN).any()) or bool((t > _WMH_T_MAX).any()):
            raise ValueError("weighted MinHash t values must be in [-2^31, 2^31 - 1]")
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.int64))   # in range: exact
    x = x.to(device=dev, dtype=torch.int64)
    k, t = x[..., 0], x[..., 1]
    k = k - ((k >> 31) << 32)                       # the uint32 bit pattern as an int32 value
    return torch.stack([k, t], dim=-1).to(torch.int32).reshape(x.shape[0], 2 * sample_size).contiguous()


def _check_topk(k) -> int:
    """``k`` of ``query_topk`` / ``neighbors``: an integer in [1, 32] (the entries one warp holds), else ``ValueError``."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= 32:
        raise ValueError("k must be an integer in [1, 32], got %r" % (k,))
    return int(k)


def _jaccard_min_count(min_jaccard: Optional[float], num_perm: int) -> int:
    """The smallest count c in 0..num_perm with ``float(c) / float(num_perm) >= min_jaccard`` -- exactly the pairs
    ``MinHash.jaccard(...) >= min_jaccard`` keeps (minhash.py:324 divides in float64 the same way; so does
    ``WeightedMinHash.jaccard``, weighted_minhash.py:60, with num_perm = the sample size).  None -> 0."""
    if min_jaccard is None:
        return 0
    t = float(min_jaccard)
    if not 0.0 <= t <= 1.0:
        raise ValueError("min_jaccard must be in [0.0, 1.0]")
    return next(c for c in range(num_perm + 1) if float(c) / float(num_perm) >= t)   # c = num_perm always qualifies
