"""Raw UTF-8 text to MinHash signatures, with word or character n-gram shingles built on the device (DESIGN.md §4m).

``shingles`` is the definition, in plain Python, as ``hashfunc.py`` holds the single-token definitions of the hash
kernels.  ``signatures`` gives, for every document, exactly
``MinHash.bulk([shingles(text, n, unit)], ...)[0].hashvalues``: the text is segmented, checked and hashed by
``dsk_shingle_count`` / ``dsk_shingle_hash`` and signed by ``dsk_minhash_bulk_ws``, so Python touches each document once
and never a shingle.  ``MinHash.bulk_text`` wraps it into MinHash objects.
"""
from __future__ import annotations

import numpy as np

from . import _native as nv
from . import engine
from .hashfunc import DEVICE_HASHES, sha1_hash32

UNITS = {"word": 0, "char": 1}      # DSK_SHINGLE_WORD, DSK_SHINGLE_CHAR
INVALID_UTF8, BAD_OFFSETS = 1, 2    # DSK_SHINGLE_INVALID_UTF8, DSK_SHINGLE_BAD_OFFSETS


def shingles(text, n=1, unit="word"):
    """The shingles of one document as UTF-8 byte strings: word n-grams (``str.split()`` words joined by one space) or
    character n-grams (code points).  A document with 1 <= m < n units gives one shingle of all of them; an empty or
    whitespace-only one gives none.  Bytes are decoded strictly (UnicodeDecodeError on malformed UTF-8)."""
    if isinstance(text, (bytes, bytearray, memoryview)):
        text = bytes(text).decode("utf-8")          # strict: UnicodeDecodeError on malformed input
    units = text.split() if unit == "word" else text  # "char": Unicode code points
    sep = " " if unit == "word" else ""
    m = len(units)
    return [sep.join(units[i:i + n]).encode("utf-8") for i in range(max(m - n + 1, min(m, 1)))]


def _hash_kind(n, unit, hashfunc) -> int:
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError("n must be an integer >= 1 (got %r)" % (n,))
    if unit not in UNITS:
        raise ValueError('unit must be "word" or "char" (got %r)' % (unit,))
    try:
        route = DEVICE_HASHES.get(hashfunc)
    except TypeError:   # an unhashable callable
        route = None
    if route is None:
        raise ValueError("signatures() hashes shingles on the device, with sha1_hash32, xxh32_hash32 or murmur3_hash32 "
                         "only; for another hashfunc use MinHash.bulk([shingles(t, n, unit) for t in texts], hashfunc=...)")
    return route[1]


def _device_text(texts):
    """(d_text, d_offsets) of CUDA tensors, or None when ``texts`` is a sequence of documents."""
    if not (isinstance(texts, tuple) and len(texts) == 2):
        return None
    import torch
    d_text, d_off = texts
    if not (isinstance(d_text, torch.Tensor) and isinstance(d_off, torch.Tensor)):
        return None
    if not (d_text.is_cuda and d_off.is_cuda and d_text.device == d_off.device):
        raise ValueError("(d_text, d_offsets) must both be CUDA tensors on one device")
    if d_text.dtype != torch.uint8 or d_text.dim() != 1 or not d_text.is_contiguous():
        raise ValueError("d_text must be a contiguous 1-D uint8 CUDA tensor")
    if d_off.dtype != torch.int64 or d_off.dim() != 1 or d_off.numel() < 1 or not d_off.is_contiguous():
        raise ValueError("d_offsets must be a contiguous 1-D int64 CUDA tensor of n_docs + 1 offsets")
    return d_text, d_off


def _host_text(texts, device: int):
    """Encodes a sequence of str / bytes-like documents back to back: (d_text, d_offsets, the encoded documents)."""
    import torch
    parts = []
    for t in texts:
        if isinstance(t, str):
            parts.append(t.encode("utf-8"))        # UnicodeEncodeError on a lone surrogate, as shingles() raises
        elif isinstance(t, (bytes, bytearray)):
            parts.append(t)
        elif isinstance(t, memoryview):
            parts.append(t.tobytes())
        else:
            raise TypeError("each document must be a str or a bytes-like object, got %s" % type(t).__name__)
    lens = np.fromiter(map(len, parts), dtype=np.int64, count=len(parts))
    off = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    blob = bytearray().join(parts)
    dev = torch.device("cuda", device)
    d_text = (torch.frombuffer(blob, dtype=torch.uint8) if len(blob) else torch.zeros(1, dtype=torch.uint8)).to(dev)
    return d_text[:len(blob)], torch.from_numpy(off).to(dev), parts


def signatures(texts, n=1, unit="word", num_perm=128, seed=1, hashfunc=sha1_hash32, permutations=None, device=0,
               to_host=True):
    """MinHash signatures of raw text documents, shingled on the device.

    ``texts`` is a sequence of ``str`` (encoded as UTF-8), a sequence of bytes-like objects, or a pair
    ``(d_text, d_offsets)`` of CUDA tensors (uint8 text, int64 offsets of its n_docs + 1 document boundaries).  Row i is
    ``MinHash.bulk([shingles(texts[i], n, unit)], num_perm=num_perm, seed=seed, hashfunc=hashfunc,
    permutations=permutations)[0].hashvalues``.  Returns that [N, K] uint64 matrix, or with ``to_host=False`` the CUDA
    int32 [N, K] tensor ``GpuLSH.insert`` / ``query_*`` / ``insert_unique`` take, without a copy to the host.

    ``hashfunc`` is one of ``sha1_hash32`` (the default), ``xxh32_hash32``, ``murmur3_hash32``.  Malformed UTF-8 raises the
    UnicodeDecodeError that decoding the lowest-numbered malformed document raises; offsets that decrease or leave the
    text raise ValueError.  One small read-back per call sizes the token buffer."""
    import torch
    kind = _hash_kind(n, unit, hashfunc)
    if permutations is None:
        from .minhash import _make_permutations
        perms = _make_permutations(num_perm, seed)
    else:
        perms = np.ascontiguousarray(np.asarray(permutations, dtype=np.uint64))
    k = perms.shape[1]
    on_device = _device_text(texts)
    if on_device is not None:
        d_text, d_off = on_device
        parts = None
        device = d_text.device.index
    else:
        nv.require_device(device)
        d_text, d_off, parts = _host_text(texts, device)
    dev = torch.device("cuda", device)
    n_docs, n_bytes = d_off.numel() - 1, d_text.numel()
    if n_docs == 0:
        return np.zeros((0, k), dtype=np.uint64) if to_host else torch.empty((0, k), dtype=torch.int32, device=dev)
    lib = nv.load()
    text_p = d_text.data_ptr() if n_bytes else None
    with torch.cuda.device(device):
        st = torch.cuda.current_stream(dev).cuda_stream
        ws_bytes = int(lib.dsk_shingle_workspace_size(n_docs, n_bytes))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        tok_off = torch.empty((n_docs + 1,), dtype=torch.int64, device=dev)
        status = torch.empty((n_docs + 1,), dtype=torch.int32, device=dev)
        nv.check(lib.dsk_shingle_count(text_p, d_off.data_ptr(), n_docs, n_bytes, UNITS[unit], int(n), tok_off.data_ptr(),
                                       status.data_ptr(), ws.data_ptr(), ws_bytes, st))
        total, summary = torch.stack([tok_off[n_docs], status[n_docs].to(torch.int64)]).tolist()
        if summary & BAD_OFFSETS:
            raise ValueError("document offsets must be non-decreasing and lie inside the text "
                             "(0 <= d_offsets[0] <= ... <= d_offsets[-1] <= len(d_text))")
        if summary & INVALID_UTF8:
            d = int(torch.nonzero(status[:n_docs])[0, 0])
            if parts is not None:
                doc = bytes(parts[d])
            else:
                a, b = d_off[d:d + 2].tolist()
                doc = d_text[a:b].cpu().numpy().tobytes()
            doc.decode("utf-8")
            raise RuntimeError("dsk_shingle_count marked document %d as malformed UTF-8, but it decodes" % d)
        tokens = torch.empty((max(total, 4),), dtype=torch.int32, device=dev)
        nv.check(lib.dsk_shingle_hash(text_p, d_off.data_ptr(), n_docs, n_bytes, UNITS[unit], int(n), kind, 0,
                                      tok_off.data_ptr(), tokens.data_ptr(), ws.data_ptr(), ws_bytes, st))
        out = engine.bulk_signatures_device(tokens, tok_off, total, perms)
    if to_host:
        return out.cpu().numpy().view(np.uint32).astype(np.uint64)
    return out
