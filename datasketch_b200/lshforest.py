"""MinHashLSHForest with the reference's API (datasketch/lshforest.py:9-186) -- a "next" row of
SURVEY.md section 8(f).  Two layers, like ``lsh.py``:

* ``MinHashLSHForest`` -- the drop-in class: l prefix "trees" kept as sorted lists of big-endian band
  keys with dict buckets, ``add / index / query / get_minhash_hashvalues / is_empty / __contains__``.
  ``add_batch`` builds the keys of a whole signature matrix with one kernel (``dsk_band_keys`` with
  b = l, r = k; the keys are byte-identical to ``_H``, lshforest.py:178-179).
* ``GpuLSHForest`` -- device-resident: per tree the documents are ordered by (k-tuple, insertion
  number); ``query`` walks prefixes r = k..1 and trees 0..l-1 exactly in the reference's order
  (lshforest.py:74-128) with a binary search on the tuples themselves, so it returns the same key
  sets for the same insertion order.
"""
from __future__ import annotations

import ctypes
from collections import defaultdict
from typing import Hashable, List, Optional, Sequence

import numpy as np

from . import _native as nv
from . import codec


class MinHashLSHForest:
    """Top-k MinHash LSH Forest (lshforest.py:9-44)."""

    def __init__(self, num_perm: int = 128, l: int = 8) -> None:
        if l <= 0 or num_perm <= 0:
            raise ValueError("num_perm and l must be positive")
        if l > num_perm:
            raise ValueError("l cannot be greater than num_perm")
        self.l = l
        self.k = int(num_perm / l)
        self.hashtables = [defaultdict(list) for _ in range(self.l)]
        self.hashranges = [(i * self.k, (i + 1) * self.k) for i in range(self.l)]
        self.keys = dict()
        self.sorted_hashtables = [[] for _ in range(self.l)]

    def _H(self, hs) -> bytes:
        return bytes(np.asarray(hs).byteswap().data)

    def _store(self, key, Hs) -> None:
        self.keys[key] = Hs
        for H, hashtable in zip(Hs, self.hashtables):
            hashtable[H].append(key)

    def add(self, key: Hashable, minhash) -> None:
        """lshforest.py:46-66 (not searchable until :meth:`index`)."""
        if len(minhash) < self.k * self.l:
            raise ValueError("The num_perm of MinHash out of range")
        if key in self.keys:
            raise ValueError("The given key has already been added")
        hv = minhash.hashvalues
        self._store(key, [self._H(hv[start:end]) for start, end in self.hashranges])

    def add_batch(self, keys: Sequence[Hashable], signatures) -> None:
        """Add many documents; all l*N band keys come from one ``dsk_band_keys`` launch."""
        from .lsh import _signature_matrix
        sig = _signature_matrix(signatures)
        if len(keys) != len(sig):
            raise ValueError("keys and signatures differ in length")
        if len(sig) == 0:
            return
        if sig.shape[1] < self.k * self.l:
            raise ValueError("The num_perm of MinHash out of range")
        seen = set()
        for key in keys:
            if key in self.keys or key in seen:
                raise ValueError("The given key has already been added")
            seen.add(key)
        width = 8 * self.k
        raw = codec.band_keys(sig, self.l, self.k).cpu().numpy().reshape(len(sig), self.l * width).tobytes()
        row = self.l * width
        for i, key in enumerate(keys):
            base = i * row
            self._store(key, [raw[base + j * width: base + (j + 1) * width] for j in range(self.l)])

    def index(self) -> None:
        """lshforest.py:68-72."""
        for i, hashtable in enumerate(self.hashtables):
            self.sorted_hashtables[i] = sorted(hashtable)

    def _query(self, minhash, r: int, b: int):
        if r > self.k or r <= 0 or b > self.l or b <= 0:
            raise ValueError("parameter outside range")
        hv = minhash.hashvalues
        hps = [self._H(hv[start: start + r]) for start, _ in self.hashranges]
        prefix_size = len(hps[0])
        for ht, hp, hashtable in zip(self.sorted_hashtables, hps, self.hashtables):
            i = self._binary_search(len(ht), lambda x, ht=ht, hp=hp: ht[x][:prefix_size] >= hp)
            if i < len(ht) and ht[i][:prefix_size] == hp:
                j = i
                while j < len(ht) and ht[j][:prefix_size] == hp:
                    for key in hashtable[ht[j]]:
                        yield key
                    j += 1

    def query(self, minhash, k: int) -> list:
        """At most k keys, longest matching prefixes first (lshforest.py:92-128)."""
        if k <= 0:
            raise ValueError("k must be positive")
        if len(minhash) < self.k * self.l:
            raise ValueError("The num_perm of MinHash out of range")
        results = set()
        r = self.k
        while r > 0:
            for key in self._query(minhash, r, self.l):
                results.add(key)
                if len(results) >= k:
                    return list(results)
            r -= 1
        return list(results)

    def get_minhash_hashvalues(self, key: Hashable) -> np.ndarray:
        """lshforest.py:130-155: rebuild the (l*k) hash values from the stored big-endian keys."""
        byteslist = self.keys.get(key, None)
        if byteslist is None:
            raise KeyError(f"The provided key does not exist in the LSHForest: {key}")
        per = len(byteslist[0]) // 8
        out = np.empty(len(byteslist) * per, dtype=np.uint64)
        for i, item in enumerate(byteslist):
            out[i * per:(i + 1) * per] = np.frombuffer(item, dtype=np.uint64).byteswap()
        return out

    def _binary_search(self, n: int, func) -> int:
        i, j = 0, n
        while i < j:
            h = int(i + (j - i) / 2)
            if not func(h):
                i = h + 1
            else:
                j = h
        return i

    def is_empty(self) -> bool:
        return any(len(t) == 0 for t in self.sorted_hashtables)

    def __contains__(self, key: Hashable) -> bool:
        return key in self.keys


class GpuLSHForest:
    """Device-resident LSH Forest over whole signature matrices.

    ``add`` appends signatures (documents are numbered in insertion order; ``keys`` optionally maps
    numbers to user keys), ``index`` sorts every tree, ``query`` returns for each query row the same
    document set ``MinHashLSHForest.query`` returns for the same insertion order.  ``query_topk`` and
    ``neighbors`` rank the documents a walk collects by Jaccard similarity on the device.

    ``weighted=True`` indexes weighted MinHash signatures, as ``MinHashLSHForest(num_perm=ss)`` does with
    ``WeightedMinHash`` objects: ``num_perm`` is the sample size ss, ``l`` and the prefix length ``k`` count samples,
    and every method that takes signatures takes ``[N, ss, 2]`` integer ``(k, t)`` rows (a numpy array, a CUDA tensor
    as ``WeightedMinHashGenerator.minhash_batch(..., to_host=False)`` returns it, or a list of ``WeightedMinHash``) with
    ``0 <= k < 2^32`` and ``-2^31 <= t < 2^31``.  The rows are held packed as ``GpuLSH(weighted=True)`` holds them
    (sample j = word 2j = k, word 2j + 1 = t); compared as unsigned words they sort like the reference's keys, so the
    query sets are the reference's.
    """

    def __init__(self, num_perm: int = 128, l: int = 8, device: int = 0, weighted: bool = False):
        if l <= 0 or num_perm <= 0:
            raise ValueError("num_perm and l must be positive")
        if l > num_perm:
            raise ValueError("l cannot be greater than num_perm")
        nv.require_device(device)
        self.l, self.k, self.h = l, int(num_perm / l), num_perm
        self.weighted = bool(weighted)
        self.sw = 2 if self.weighted else 1          # words per sample
        self.device = device
        self._blocks: List = []
        self._sig = None
        self._order = None
        self.keys: List[Hashable] = []

    def __len__(self) -> int:
        return sum(int(b.shape[0]) for b in self._blocks)

    def _dev_sig(self, sig):
        import torch
        from .lsh import _pack_weighted, _signature_matrix
        if self.weighted:
            return _pack_weighted(sig, self.h, torch.device("cuda", self.device))
        if isinstance(sig, np.ndarray):
            sig = torch.from_numpy(_signature_matrix(sig).view(np.int32)).cuda(self.device)
        if sig.dim() != 2 or sig.shape[1] < self.k * self.l or sig.shape[1] != self.h:
            raise ValueError("The num_perm of MinHash out of range")
        if sig.element_size() != 4:
            raise TypeError("GpuLSHForest takes the 32-bit signature matrix")
        return sig.contiguous()

    def add(self, sig, keys: Optional[Sequence[Hashable]] = None) -> None:
        self._blocks.append(self._dev_sig(sig))
        if keys is not None:
            self.keys.extend(keys)

    def is_empty(self) -> bool:
        return self._order is None or self._order.shape[1] == 0

    def index(self) -> None:
        """Sort every tree by (k-tuple, document number): stable LSD passes over pairs of columns
        (``torch.sort`` is used as the sort primitive; the query walk is the hand-written kernel).  On a weighted
        forest a tree spans 2k words and each pair of columns is one ``(k, t)`` sample."""
        import torch
        width = self.sw * self.h
        self._sig = torch.cat(self._blocks, 0) if self._blocks else torch.zeros((0, width), dtype=torch.int32,
                                                                             device=torch.device("cuda", self.device))
        self._blocks = [self._sig] if len(self._sig) else []
        n = self._sig.shape[0]
        u = self._sig.to(torch.int64) & 0xFFFFFFFF
        kw = self.sw * self.k                        # words per tree
        orders = []
        for t in range(self.l):
            order = torch.arange(n, device=self._sig.device)
            cols = list(range(t * kw, (t + 1) * kw))
            while cols:
                hi_lo = cols[-2:]
                cols = cols[:-2]
                if len(hi_lo) == 2:
                    key = (u[order, hi_lo[0]] << 32 | u[order, hi_lo[1]]) - (1 << 63)   # unsigned order as signed
                else:
                    key = u[order, hi_lo[0]]
                order = order[torch.sort(key, stable=True).indices]
            orders.append(order.to(torch.int32))
        self._order = torch.stack(orders) if orders else None

    def _indexed(self):
        if self._order is None:
            raise ValueError("index() has not been called")
        n = self._sig.shape[0]
        return (self._sig.data_ptr() if n else None), (self._order.data_ptr() if n else None), n

    def query(self, sig, k: int, to_host: bool = True):
        """[Q, K] query signatures -> int32 [Q, k] document numbers (-1 pads), per row the set the
        reference's ``query(minhash, k)`` returns."""
        import torch
        if k <= 0:
            raise ValueError("k must be positive")
        d_sig, d_order, n = self._indexed()
        sig = self._dev_sig(sig)
        nq = sig.shape[0]
        out = torch.empty((nq, k), dtype=torch.int32, device=sig.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            if self.weighted:
                nv.check(nv.load().dsk_forest_query_weighted(d_sig, d_order, n, self.h, self.l, self.k, sig.data_ptr(), nq,
                                                             k, out.data_ptr(), st))
            else:
                nv.check(nv.load().dsk_forest_query(d_sig, d_order, n, self.h, self.l, self.k, sig.data_ptr(), nq, k,
                                                    out.data_ptr(), st))
        return out.cpu().numpy() if to_host else out

    def query_keys(self, sig, k: int) -> List[list]:
        res = self.query(sig, k)
        return [[(self.keys[i] if self.keys else int(i)) for i in row if i >= 0] for row in res]

    # -- ranked answers: the reference docstring's post-processing, on the device -------------------------------------
    @staticmethod
    def _check_candidates(candidates, k: int) -> int:
        if candidates is None:
            candidates = 2 * k
        if isinstance(candidates, bool) or not isinstance(candidates, (int, np.integer)) or not k <= candidates <= 1024:
            raise ValueError("candidates must be an integer in [k, 1024], got %r" % (candidates,))
        return int(candidates)

    def query_topk(self, sig, k: int, candidates: Optional[int] = None, min_jaccard: Optional[float] = None,
                   to_host: bool = True):
        """Each query's k most similar documents among its forest candidates: ``(idx int32[Q, k], eq int32[Q, k])``.

        The reference's ``query`` docstring suggests asking for a multiple of k and keeping the k best by Jaccard
        similarity; this does that on the device.  For query m, row q is::

            cand = forest.query(m, candidates)          # the set query(sig, candidates) returns
            sorted([d for d in cand if m.jaccard(doc[d]) >= t], key=lambda d: (-m.jaccard(doc[d]), d))[:k]

        with -1 / -1 behind the list.  ``eq`` counts the equal positions over all ``num_perm`` (on a weighted forest:
        the samples whose whole ``(k, t)`` pairs agree), so ``eq / num_perm`` is ``MinHash.jaccard`` /
        ``WeightedMinHash.jaccard``; columns past ``l * k``, which the walk never reads, count too.  ``k`` is in
        ``[1, 32]``, ``candidates`` (default ``2 * k``) in ``[k, 1024]``.  ``min_jaccard`` only removes documents from
        the collected set; it never changes which are collected.  One launch, no host synchronisation, and an output
        of ``Q * k`` entries."""
        import torch
        from .lsh import _check_topk, _jaccard_min_count
        k = _check_topk(k)
        candidates = self._check_candidates(candidates, k)
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_sig, d_order, n = self._indexed()
        sig = self._dev_sig(sig)
        nq = sig.shape[0]
        with torch.cuda.device(self.device):
            idx = torch.empty((max(nq, 1), k), dtype=torch.int32, device=sig.device)
            eq = torch.empty((max(nq, 1), k), dtype=torch.int32, device=sig.device)
            nv.check(nv.load().dsk_forest_query_topk(d_sig, d_order, n, self.h, int(self.weighted), self.l, self.k,
                                                     sig.data_ptr() if nq else None, nq, candidates, mc, k,
                                                     idx.data_ptr(), eq.data_ptr(), torch.cuda.current_stream().cuda_stream))
            idx, eq = idx[:nq], eq[:nq]
        if to_host:
            return idx.cpu().numpy(), eq.cpu().numpy()
        return idx, eq

    def neighbors(self, k: int, candidates: Optional[int] = None, min_jaccard: Optional[float] = None,
                  to_host: bool = True):
        """The k nearest neighbours of every indexed document, with no LSH threshold: ``(idx int32[n, k], eq int32[n, k])``.

        Row i ranks, as ``query_topk`` does, the first ``candidates`` distinct documents other than i that the forest
        walk of document i's own row meets -- in reference terms::

            res = set()
            for r in range(forest.k, 0, -1):
                for d in forest._query(doc[i], r, forest.l):
                    if d != i: res.add(d)
                    if len(res) >= candidates: stop both loops

        The test is by document number, so an exact copy of i stays a neighbour.  One launch, no host synchronisation."""
        import torch
        from .lsh import _check_topk, _jaccard_min_count
        k = _check_topk(k)
        candidates = self._check_candidates(candidates, k)
        mc = _jaccard_min_count(min_jaccard, self.h)
        d_sig, d_order, n = self._indexed()
        with torch.cuda.device(self.device):
            dev = torch.device("cuda", self.device)
            idx = torch.empty((max(n, 1), k), dtype=torch.int32, device=dev)
            eq = torch.empty((max(n, 1), k), dtype=torch.int32, device=dev)
            nv.check(nv.load().dsk_forest_neighbors(d_sig, d_order, n, self.h, int(self.weighted), self.l, self.k,
                                                    candidates, mc, k, idx.data_ptr(), eq.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
            idx, eq = idx[:n], eq[:n]
        if to_host:
            return idx.cpu().numpy(), eq.cpu().numpy()
        return idx, eq
