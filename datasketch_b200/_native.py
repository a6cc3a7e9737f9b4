"""ctypes binding of libdsk_b200.so (include/dsk.h).

The shared library is the product; this module only loads it and maps its
return codes onto the exception types the reference raises.  There is no CPU
fallback anywhere: if the library cannot be loaded the import fails loudly, and
if no H100 is present every compute entry point raises RuntimeError -- the same
exception the reference raises for ``gpu_mode='always'`` without a device
(datasketch/minhash.py:272-274).
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional

import numpy as np

from . import _build

_HERE = os.path.dirname(os.path.abspath(__file__))

DSK_OK, DSK_ERR_INVALID, DSK_ERR_CUDA, DSK_ERR_NO_DEVICE, DSK_ERR_ALIGN, DSK_ERR_NOMEM = range(6)
KERNEL_AUTO, KERNEL_TWO_PHASE, KERNEL_DIRECT, KERNEL_EXACT = range(4)

c_void_p, c_int, c_int64, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t

# every symbol include/dsk.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "dsk_version": (c_int, []),
    "dsk_last_error": (ctypes.c_char_p, []),
    "dsk_device_count": (c_int, []),
    "dsk_device_info": (c_int, [c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int),
                                ctypes.POINTER(c_size_t)]),
    "dsk_perm_create": (c_int, [c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "dsk_perm_info": (c_int, [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "dsk_perm_destroy": (None, [c_void_p]),
    "dsk_perm_analyze": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "dsk_minhash_bulk": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int,
                                 c_void_p, c_int, c_int, c_void_p]),
    "dsk_minhash_bulk_workspace_size": (ctypes.c_size_t, [c_int64, c_int64]),
    "dsk_minhash_bulk_ws": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int,
                                    c_void_p, c_int, c_int, c_void_p, ctypes.c_size_t, c_void_p]),
    "dsk_minhash_bulk_gather": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p, c_int,
                                        c_int64, c_int, c_int, c_void_p]),
    "dsk_minhash_bulk_host": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int64, c_void_p, c_int64, c_int,
                                      c_void_p, c_int, c_int]),
    "dsk_release_host_pipeline": (c_int, [c_int]),
    "dsk_sig_merge_min": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "dsk_wmh_create": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "dsk_wmh_destroy": (None, [c_void_p]),
    "dsk_wmh_minhash": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_void_p]),
    "dsk_wmh_minhash_csr": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int,
                                    c_void_p]),
    "dsk_lsh_create": (c_int, [c_int, c_int, c_int, c_int64, c_int, ctypes.POINTER(c_void_p)]),
    "dsk_lsh_create_weighted": (c_int, [c_int, c_int, c_int, c_int64, c_int, ctypes.POINTER(c_void_p)]),
    "dsk_lsh_destroy": (None, [c_void_p]),
    "dsk_lsh_size": (c_int, [c_void_p, ctypes.POINTER(c_int64), ctypes.POINTER(c_int64)]),
    "dsk_lsh_insert": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "dsk_lsh_insert_tokens": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p]),
    "dsk_lsh_query_count": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "dsk_lsh_query_fill": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "dsk_exclusive_scan": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_pairs_count": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "dsk_lsh_pairs_fill": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_clusters": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "dsk_lsh_query_jaccard_count": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "dsk_lsh_query_jaccard_fill": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_query_best": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_query_topk": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_neighbors": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_unique_workspace_size": (ctypes.c_size_t, [c_void_p, c_int64]),
    "dsk_lsh_unique_count": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "dsk_lsh_unique_commit": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(c_int64), c_void_p]),
    "dsk_lsh_ensemble_create": (c_int, [c_int, c_int, c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(c_void_p)]),
    "dsk_lsh_ensemble_destroy": (None, [c_void_p]),
    "dsk_lsh_ensemble_size": (c_int, [c_void_p, ctypes.POINTER(c_int64)]),
    "dsk_lsh_ensemble_index_bytes": (ctypes.c_size_t, [c_void_p, c_int64]),
    "dsk_lsh_ensemble_index": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_query_count": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_query_fill": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_containment_count": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, ctypes.c_double,
                                                   c_void_p, c_void_p]),
    "dsk_lsh_ensemble_containment_fill": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, ctypes.c_double,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_containment_topk": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, ctypes.c_double,
                                                  c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_self_containment_count": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_double, c_void_p, c_void_p]),
    "dsk_lsh_ensemble_self_containment_fill": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_double, c_void_p, c_void_p,
                                                       c_void_p, c_void_p, c_void_p]),
    "dsk_ensemble_partition_workspace_size": (ctypes.c_size_t, [c_int64, c_int]),
    "dsk_ensemble_partition": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, ctypes.c_size_t, c_int, c_void_p,
                                       c_void_p, c_void_p]),
    "dsk_lsh_remove": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "dsk_lsh_alive": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "dsk_lsh_compact_workspace_size": (ctypes.c_size_t, [c_void_p]),
    "dsk_lsh_compact": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_size_t, c_void_p]),
    "dsk_jaccard_pairs": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "dsk_jaccard_topk": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    "dsk_jaccard_topk_workspace_size": (ctypes.c_size_t, [c_int64, c_int64, c_int]),
    "dsk_jaccard_topk_ws": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p,
                                    ctypes.c_size_t, c_void_p]),
    "dsk_sha1_tokens": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int, c_void_p]),
    "dsk_hash_tokens": (c_int, [c_void_p, c_void_p, c_int64, c_int, ctypes.c_uint32, c_void_p, c_void_p]),
    "dsk_shingle_workspace_size": (c_size_t, [c_int64, c_int64]),
    "dsk_shingle_count": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t,
                                  c_void_p]),
    "dsk_shingle_hash": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, ctypes.c_uint32, c_void_p,
                                 c_void_p, c_void_p, c_size_t, c_void_p]),
    "dsk_bbit_pack": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "dsk_bbit_unpack": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "dsk_forest_query": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_int, c_void_p,
                                 c_void_p]),
    "dsk_forest_query_weighted": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_int,
                                          c_void_p, c_void_p]),
    "dsk_forest_query_topk": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_int,
                                      c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dsk_forest_neighbors": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p]),
    "dsk_lean_pack": (c_int, [c_void_p, c_int, c_int64, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "dsk_lean_unpack": (c_int, [c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "dsk_band_keys": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dsk_band_fingerprints": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dsk_band_sums": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dsk_bloom_insert": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_int,
                                 c_void_p]),
    "dsk_bloom_query": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_int,
                                c_void_p, c_void_p]),
    "dsk_bloom_unique_workspace_size": (c_size_t, [c_int64, c_int, c_int, c_int, c_int]),
    "dsk_bloom_unique": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_int,
                                 c_void_p, c_size_t, c_void_p, c_void_p]),
}

_lib = None
_lock = threading.Lock()


def lib_path() -> str:
    return _build.LIB


def load():
    """Load (building first if the sources are newer and nvcc exists) the native library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = _build.LIB
        if _build._stale() and (_build.have_nvcc() or not os.path.exists(path)):
            try:
                _build.build()
            except Exception as exc:  # noqa: BLE001
                raise RuntimeError(
                    "datasketch_b200: libdsk_b200.so is missing/stale and could not be built (%s). "
                    "This package has no CPU fallback." % exc) from exc
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError here = header/library drift: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error() -> str:
    msg = load().dsk_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int) -> None:
    if rc == DSK_OK:
        return
    msg = last_error()
    if rc in (DSK_ERR_INVALID, DSK_ERR_ALIGN):
        raise ValueError(msg)
    if rc == DSK_ERR_NOMEM:
        raise MemoryError(msg)
    if rc == DSK_ERR_NO_DEVICE:
        raise RuntimeError("H100 GPU required but unavailable (no CPU fallback): " + msg)
    raise RuntimeError(msg)


def device_count() -> int:
    return int(load().dsk_device_count())


def require_device(device: int = 0) -> None:
    if device_count() <= device:
        raise RuntimeError("H100 GPU required but CUDA device %d is unavailable (no CPU fallback)." % device)


def device_info(device: int = 0) -> dict:
    sm, ma, mi, mem = c_int(), c_int(), c_int(), c_size_t()
    check(load().dsk_device_info(device, ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi), ctypes.byref(mem)))
    return {"sm_count": sm.value, "cc": (ma.value, mi.value), "total_mem": mem.value}


def ptr(x) -> Optional[int]:
    """Raw address of a numpy array (host) or torch tensor (device or host)."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    return x.data_ptr()


def perm_analyze(permutations: np.ndarray) -> np.ndarray:
    """Host-only: bool[K], True where the fast kernels would not be exact for 32-bit tokens."""
    perms = np.ascontiguousarray(permutations, dtype=np.uint64)
    a, b = np.ascontiguousarray(perms[0]), np.ascontiguousarray(perms[1])
    out = np.zeros(perms.shape[1], dtype=np.uint8)
    load().dsk_perm_analyze(a.ctypes.data, b.ctypes.data, int(perms.shape[1]), out.ctypes.data)
    return out.astype(bool)


class PermHandle:
    """Owns a ``dsk_perm*`` (device copy + safety analysis of one permutation set)."""

    def __init__(self, permutations: np.ndarray, device: int = 0):
        perms = np.ascontiguousarray(permutations, dtype=np.uint64)
        if perms.ndim != 2 or perms.shape[0] != 2:
            raise ValueError("permutations must have shape (2, num_perm)")
        self.num_perm = int(perms.shape[1])
        self.device = device
        h = c_void_p()
        a = np.ascontiguousarray(perms[0])
        b = np.ascontiguousarray(perms[1])
        check(load().dsk_perm_create(a.ctypes.data, b.ctypes.data, self.num_perm, device, ctypes.byref(h)))
        self._h = h
        n, bad, dev = c_int(), c_int(), c_int()
        check(load().dsk_perm_info(self._h, ctypes.byref(n), ctypes.byref(bad), ctypes.byref(dev)))
        self.n_unsafe = bad.value

    @property
    def handle(self):
        return self._h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and _lib is not None:
                _lib.dsk_perm_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass


_perm_cache: dict = {}
_perm_cache_lock = threading.Lock()


def perm_handle(permutations: np.ndarray, device: int = 0) -> PermHandle:
    """Cached PermHandle keyed by the permutation bytes (a few KB)."""
    perms = np.ascontiguousarray(permutations, dtype=np.uint64)
    key = (device, perms.shape[1], perms.tobytes())
    with _perm_cache_lock:
        h = _perm_cache.get(key)
        if h is None:
            if len(_perm_cache) > 64:
                _perm_cache.clear()
            h = PermHandle(perms, device)
            _perm_cache[key] = h
    return h
