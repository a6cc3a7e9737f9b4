"""MinHash with the reference's API surface, computed on the H100.

Mirrors ``datasketch.MinHash`` (datasketch/minhash.py:51-537): same constructor
arguments, attributes (``seed``, ``num_perm``, ``hashfunc``, ``hashvalues``
np.uint64[K], ``permutations`` (2, K) np.uint64), methods and exceptions.  What
differs is *where the arithmetic runs*: ``update`` / ``update_batch`` only hash
the tokens on the host (the reference's contract, minhash.py:85-87, :262-263)
and queue the integer hash values; the permutation-hash-and-min
(minhash.py:221-224, :294-297) runs in ``libdsk_b200.so`` when the state is
next observed (``hashvalues``, ``jaccard``, ``merge`` ...), one fused kernel over
everything queued.  ``bulk`` / ``generator`` send the whole batch in one call.

There is no CPU path.  ``gpu_mode`` is accepted for signature compatibility;
whatever its value, a missing H100 raises the RuntimeError the reference raises
for ``gpu_mode='always'`` (minhash.py:272-274).
"""
from __future__ import annotations

import copy
import gc
import warnings
from typing import Callable, Generator, Iterable, List, Optional

import numpy as np

from . import engine
from .hashfunc import DEVICE_HASHES, sha1_hash32

# minhash.py:27, :30-32
hashvalue_byte_size = len(bytes(np.int64(42).data))
_mersenne_prime = np.uint64((1 << 61) - 1)
_max_hash = np.uint64((1 << 32) - 1)
_hash_range = 1 << 32

_GPU_MODES = ("disable", "detect", "always")


def _make_permutations(num_perm: int, seed: int) -> np.ndarray:
    """Host-side parameter generation, bit-identical to minhash.py:170-184.

    Row 0 = a in [1, p), row 1 = b in [0, p), drawn interleaved (a0, b0, a1, b1, ...)
    from one ``RandomState(seed)``.  Never re-implemented on device.
    """
    gen = np.random.RandomState(seed)
    ab = np.empty((num_perm, 2), dtype=np.uint64)
    for i in range(num_perm):
        ab[i, 0] = gen.randint(1, _mersenne_prime, dtype=np.uint64)
        ab[i, 1] = gen.randint(0, _mersenne_prime, dtype=np.uint64)
    return np.ascontiguousarray(ab.T)


class MinHash:
    """MinHash sketch (see module docstring).  Args as datasketch/minhash.py:113-122."""

    def __init__(self, num_perm: int = 128, seed: int = 1, gpu_mode: str = "disable",
                 hashfunc: Callable = sha1_hash32, hashobj: Optional[object] = None,
                 hashvalues: Optional[Iterable] = None, permutations=None) -> None:
        if hashvalues is not None:
            num_perm = len(hashvalues)
        if num_perm > _hash_range:
            raise ValueError("Cannot have more than %d number of permutation functions" % _hash_range)
        self.seed = seed
        self.num_perm = num_perm
        if not callable(hashfunc):
            raise ValueError("The hashfunc must be a callable.")
        self.hashfunc = hashfunc
        if hashobj is not None:
            warnings.warn("hashobj is deprecated, use hashfunc instead.", DeprecationWarning, stacklevel=2)
        self._pending: List[int] = []
        if hashvalues is not None:
            self._state = self._parse_hashvalues(hashvalues)
        else:
            self._state = self._init_hashvalues(num_perm)
        if permutations is not None:
            self.permutations = permutations
        else:
            self.permutations = self._init_permutations(num_perm)
        if len(self._state) != len(self.permutations[0]):
            raise ValueError("Numbers of hash values and permutations mismatch")
        self._gpu_mode = gpu_mode

    # -- state ---------------------------------------------------------------------------
    def _init_hashvalues(self, num_perm: int) -> np.ndarray:
        return np.full(num_perm, _max_hash, dtype=np.uint64)

    def _init_permutations(self, num_perm: int) -> np.ndarray:
        return _make_permutations(num_perm, self.seed)

    def _parse_hashvalues(self, hashvalues) -> np.ndarray:
        return np.array(hashvalues, dtype=np.uint64)

    def _flush(self) -> None:
        """Fold every queued token hash into the state with ONE kernel launch."""
        if not self._pending:
            return
        pending, self._pending = self._pending, []
        tok, off = engine.pack_docs([pending])
        perms = np.ascontiguousarray(np.asarray(self.permutations, dtype=np.uint64))
        out = engine.bulk_signatures(tok, off, perms, init=self._state, out_u64=True)
        self._state = out[0]

    @property
    def hashvalues(self) -> np.ndarray:
        self._flush()
        return self._state

    @hashvalues.setter
    def hashvalues(self, value) -> None:
        # an assignment replaces the state that queued tokens would have been folded into
        self._pending = []
        self._state = value

    # -- updates ----------------------------------------------------------------------------
    def update(self, b) -> None:
        """Add one value (minhash.py:189-224).  Hashing is host-side; the permutation
        hash + min is deferred to the next flush."""
        self._pending.append(self.hashfunc(b))
        if len(self._pending) >= (1 << 20):
            self._flush()

    def update_batch(self, b: Iterable) -> None:
        """Add many values (minhash.py:226-297).  An empty batch is a no-op (:265-266)."""
        hv = [self.hashfunc(_b) for _b in b]
        if not hv:
            return
        engine.nv.require_device(0)  # same moment the reference raises for gpu_mode='always'
        self._pending.extend(hv)
        if len(self._pending) >= (1 << 20):
            self._flush()

    # -- estimators -----------------------------------------------------------------------------
    def jaccard(self, other: "MinHash") -> float:
        """minhash.py:299-324 (same checks, same float)."""
        if other.seed != self.seed:
            raise ValueError("Cannot compute Jaccard given MinHash with different seeds")
        if len(self) != len(other):
            raise ValueError("Cannot compute Jaccard given MinHash with different numbers of permutation functions")
        return float(np.count_nonzero(self.hashvalues == other.hashvalues)) / float(len(self))

    def count(self) -> float:
        """minhash.py:326-335."""
        k = len(self)
        return float(k) / np.sum(self.hashvalues / float(_max_hash)) - 1.0

    def merge(self, other: "MinHash") -> None:
        """minhash.py:337-359."""
        if other.seed != self.seed:
            raise ValueError("Cannot merge MinHash with different seeds")
        if len(self) != len(other):
            raise ValueError("Cannot merge MinHash with different numbers of permutation functions")
        self.hashvalues = np.minimum(other.hashvalues, self.hashvalues)

    def digest(self) -> np.ndarray:
        return copy.copy(self.hashvalues)

    def is_empty(self) -> bool:
        return not np.any(self.hashvalues != _max_hash)

    def clear(self) -> None:
        self.hashvalues = self._init_hashvalues(len(self))

    def copy(self) -> "MinHash":
        """minhash.py:385-393: state copied, permutations shared by reference."""
        return MinHash(seed=self.seed, hashfunc=self.hashfunc, hashvalues=self.digest(),
                       permutations=self.permutations, gpu_mode=self._gpu_mode)

    def __len__(self) -> int:
        return len(self._state)

    def __eq__(self, other) -> bool:
        return (type(self) is type(other) and self.seed == other.seed
                and np.array_equal(self.hashvalues, other.hashvalues))

    __hash__ = None  # same as the reference: defining __eq__ without __hash__

    @classmethod
    def union(cls, *mhs: "MinHash") -> "MinHash":
        """minhash.py:411-462."""
        if len(mhs) < 2:
            raise ValueError("Cannot union less than 2 MinHash")
        num_perm = len(mhs[0])
        seed = mhs[0].seed
        if any((seed != m.seed or num_perm != len(m)) for m in mhs):
            raise ValueError("The unioning MinHash must have the same seed and number of permutation functions")
        hashvalues = np.minimum.reduce([m.hashvalues for m in mhs])
        return cls(num_perm=num_perm, seed=seed, hashfunc=mhs[0].hashfunc, hashvalues=hashvalues,
                   permutations=mhs[0].permutations, gpu_mode=mhs[0]._gpu_mode)

    # -- bulk -----------------------------------------------------------------------------------
    @classmethod
    def _from_row(cls, proto: "MinHash", row: np.ndarray) -> "MinHash":
        m = cls.__new__(cls)
        m.seed = proto.seed
        m.num_perm = proto.num_perm
        m.hashfunc = proto.hashfunc
        m._pending = []
        m._state = row
        m.permutations = proto.permutations
        m._gpu_mode = proto._gpu_mode
        return m

    @classmethod
    def bulk(cls, b: Iterable, **minhash_kwargs) -> List["MinHash"]:
        """minhash.py:464-489.  All documents go to the GPU in one pipelined call."""
        return list(cls.generator(b, **minhash_kwargs))

    @classmethod
    def generator(cls, b: Iterable, batch_docs: int = 1 << 16, **minhash_kwargs) -> Generator["MinHash", None, None]:
        """minhash.py:491-522.  Documents are hashed on the host (``hashfunc``) and sent to the
        device ``batch_docs`` at a time; each yielded MinHash starts from the empty state and
        shares the prototype's permutations, exactly like ``m.copy()`` in the reference."""
        proto = cls(**minhash_kwargs)
        perms = np.ascontiguousarray(np.asarray(proto.permutations, dtype=np.uint64))
        hf = proto.hashfunc
        batch: list = []

        # With a hash function the library has on device (the reference's default sha1_hash32, or the xxh32 /
        # murmur3 functions of .hashfunc) hashing moves to the device too: same values, no per-token Python call.
        try:
            device_hash = DEVICE_HASHES.get(hf)
        except TypeError:  # an unhashable callable
            device_hash = None

        def run(docs):
            init = proto.hashvalues if not proto.is_empty() else None
            sig = None
            if device_hash is not None:
                try:
                    sig = engine.bulk_signatures_sha1(docs, perms, init=init, hash_kind=device_hash[1])
                except TypeError:
                    sig = None  # a non-bytes token: the per-token route below raises what the reference raises
            if sig is None:
                tok, off = engine.pack_docs([[hf(t) for t in d] for d in docs])
                sig = engine.bulk_signatures(tok, off, perms, init=init, out_u64=True)
            # One object per row.  The cyclic GC is paused for the burst: tens of thousands of fresh container
            # objects would otherwise trigger full collections that re-traverse the caller's (large) corpus.
            gc_was_on = gc.isenabled()
            gc.disable()
            try:
                out = [cls._from_row(proto, row.copy()) for row in sig]
            finally:
                if gc_was_on:
                    gc.enable()
            yield from out

        for doc in b:
            batch.append(doc if isinstance(doc, (list, tuple)) else list(doc))
            if len(batch) >= batch_docs:
                yield from run(batch)
                batch = []
        if batch:
            yield from run(batch)

    @classmethod
    def bulk_text(cls, texts, n: int = 1, unit: str = "word", **minhash_kwargs) -> List["MinHash"]:
        """One MinHash per raw text document: ``MinHash.bulk([shingles(t, n, unit) for t in texts], **minhash_kwargs)``
        with the word / character n-gram shingles built, hashed and signed on the device (``shingle.signatures``).
        ``texts`` is a sequence of ``str`` or bytes-like documents, or a ``(d_text, d_offsets)`` pair of CUDA tensors."""
        from .shingle import signatures
        proto = cls(**minhash_kwargs)
        perms = np.ascontiguousarray(np.asarray(proto.permutations, dtype=np.uint64))
        sig = signatures(texts, n, unit, seed=proto.seed, hashfunc=proto.hashfunc, permutations=perms)
        if not proto.is_empty():
            sig = np.minimum(sig, proto.hashvalues)
        return [cls._from_row(proto, row.copy()) for row in sig]

    # -- pickling: only host state travels (cf. minhash.py:529-537) ---------------------------------
    def __getstate__(self):
        self._flush()
        return {"seed": self.seed, "num_perm": self.num_perm, "hashfunc": self.hashfunc,
                "hashvalues": self._state, "permutations": self.permutations, "_gpu_mode": self._gpu_mode}

    def __setstate__(self, state):
        self.seed = state["seed"]
        self.num_perm = state["num_perm"]
        self.hashfunc = state["hashfunc"]
        self._state = state["hashvalues"]
        self._pending = []
        self.permutations = state["permutations"]
        self._gpu_mode = state.get("_gpu_mode", "disable")
