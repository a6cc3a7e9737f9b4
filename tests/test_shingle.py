"""Raw UTF-8 text to word / character n-gram shingles on the device: ``dsk_shingle_count`` / ``dsk_shingle_hash``
(shingle_kernels.cuh) and ``datasketch_b200.shingle.signatures`` / ``MinHash.bulk_text``.

The definition is ``shingle.shingles`` (the shingles of one document as UTF-8 bytes).  Most cases run twice, as in
test_wmh_sparse.py: on the emulated library through the C-ABI (CPU suite, small sizes) and on the H100 (``-m gpu``), where
the tokens come through the same C-ABI and the signatures through the Python API.  Expected tokens are the token hash of
every shingle of ``shingles()``, expected statuses ``bytes.decode`` failing, and expected signatures the reference's
``MinHash.bulk`` in tests/golden/shingles.npz (oracle/gen_golden_shingles.py) or ``MinHash.bulk`` over ``shingles()``.
"""
import numpy as np
import pytest

from datasketch_b200.hashfunc import murmur3_hash32, sha1_hash32, xxh32_hash32
from datasketch_b200.shingle import shingles
from oracle import oracle_np as o

DSK_OK, DSK_ERR_INVALID = 0, 1
WORD, CHAR = 0, 1
INVALID_UTF8, BAD_OFFSETS = 1, 2
HASHES = {0: sha1_hash32, 1: xxh32_hash32, 2: murmur3_hash32}
CONFIGS = [("word", 1), ("word", 3), ("word", 5), ("char", 1), ("char", 4), ("char", 9)]
WHITESPACE = [0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x1C, 0x1D, 0x1E, 0x1F, 0x20, 0x85, 0xA0, 0x1680] + \
    list(range(0x2000, 0x200B)) + [0x2028, 0x2029, 0x202F, 0x205F, 0x3000]


def _pack(docs):
    off = np.zeros(len(docs) + 1, dtype=np.int64)
    np.cumsum([len(d) for d in docs], out=off[1:])
    return np.frombuffer(b"".join(docs), dtype=np.uint8), off


def _want(docs, n, unit, kind=0):
    """(invalid[N], token offsets, tokens) of the definition."""
    hf = HASHES[kind]
    bad, offs, toks = [], [0], []
    for d in docs:
        try:
            sh = shingles(d, n, unit)
            bad.append(False)
        except UnicodeDecodeError:
            sh = []
            bad.append(True)
        toks.extend(hf(s) for s in sh)
        offs.append(len(toks))
    return np.array(bad, dtype=bool), np.array(offs, dtype=np.int64), np.array(toks, dtype=np.uint32)


def _fixture_docs(golden):
    g = golden("shingles")
    text, off = g["text"].tobytes(), g["offsets"]
    return g, [text[off[i]:off[i + 1]] for i in range(len(off) - 1)]


def _fixture_shingles(g, key):
    """(shingle bytes back to back, shingle offsets, per-document shingle offsets) of one configuration."""
    so = np.zeros(len(g[key + "_len"]) + 1, dtype=np.int64)
    np.cumsum(g[key + "_len"], out=so[1:])
    dp = np.zeros(len(g[key + "_count"]) + 1, dtype=np.int64)
    np.cumsum(g[key + "_count"], out=dp[1:])
    return g[key + "_bytes"].tobytes(), so, dp


class _Emu:
    """The emulated library through the C-ABI, on host buffers."""
    name = "emu"

    def __init__(self, lib):
        self.lib = lib

    def _ws(self, n_docs, n_bytes):
        nb = int(self.lib.dsk_shingle_workspace_size(n_docs, n_bytes))
        buf = np.zeros(nb // 8 + 4, dtype=np.int64)
        return buf, (buf.ctypes.data + 15) // 16 * 16, nb

    def raw(self, text, off, unit, n, kind=0, seed=0):
        """(rc of count, status[N+1], tok_off[N+1], tokens) for text (uint8) and offsets (int64) as given."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.int64)
        N = len(off) - 1
        tp = text.ctypes.data if len(text) else None
        _keep, wsp, nb = self._ws(N, len(text))
        tok_off = np.full(N + 1, -7, dtype=np.int64)
        st = np.full(N + 1, -7, dtype=np.int32)
        rc = self.lib.dsk_shingle_count(tp, off.ctypes.data, N, len(text), unit, n, tok_off.ctypes.data, st.ctypes.data,
                                        wsp, nb, None)
        if rc:
            return rc, None, None, None
        tot = int(tok_off[N])
        tok = np.zeros(max(tot, 1), dtype=np.uint32)
        rc = self.lib.dsk_shingle_hash(tp, off.ctypes.data, N, len(text), unit, n, kind, seed, tok_off.ctypes.data,
                                       tok.ctypes.data, wsp, nb, None)
        assert rc == DSK_OK, self.lib.dsk_last_error()
        return DSK_OK, st, tok_off, tok[:tot]

    def tokens(self, docs, n, unit, kind=0):
        text, off = _pack(docs)
        rc, st, tok_off, tok = self.raw(text, off, WORD if unit == "word" else CHAR, n, kind)
        assert rc == DSK_OK, self.lib.dsk_last_error()
        return st, tok_off, tok

    def sig(self, docs, n, unit, kind=0, num_perm=128):
        _, tok_off, tok = self.tokens(docs, n, unit, kind)
        return o.bulk_signatures_csr(tok, tok_off, num_perm, 1)


class _Gpu:
    """The compiled library on the H100: tokens through the C-ABI on CUDA tensors, signatures through the Python API."""
    name = "gpu"

    def __init__(self):
        import torch
        from datasketch_b200 import _native as nv
        self.torch, self.lib = torch, nv.load()

    def raw(self, text, off, unit, n, kind=0, seed=0):
        torch = self.torch
        d_text = text if isinstance(text, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(text, np.uint8).copy()).cuda()
        d_off = off if isinstance(off, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(off, np.int64)).cuda()
        N, nbytes = d_off.numel() - 1, d_text.numel()
        nb = int(self.lib.dsk_shingle_workspace_size(N, nbytes))
        ws = torch.empty(max(nb, 16), dtype=torch.uint8, device="cuda")
        tok_off = torch.full((N + 1,), -7, dtype=torch.int64, device="cuda")
        st = torch.full((N + 1,), -7, dtype=torch.int32, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        tp = d_text.data_ptr() if nbytes else None
        rc = self.lib.dsk_shingle_count(tp, d_off.data_ptr(), N, nbytes, unit, n, tok_off.data_ptr(), st.data_ptr(),
                                        ws.data_ptr(), nb, s)
        if rc:
            return rc, None, None, None
        tot = int(tok_off[N])
        tok = torch.zeros(max(tot, 1), dtype=torch.int32, device="cuda")
        rc = self.lib.dsk_shingle_hash(tp, d_off.data_ptr(), N, nbytes, unit, n, kind, seed, tok_off.data_ptr(),
                                       tok.data_ptr(), ws.data_ptr(), nb, s)
        assert rc == DSK_OK, self.lib.dsk_last_error()
        return DSK_OK, st.cpu().numpy(), tok_off.cpu().numpy(), tok[:tot].cpu().numpy().view(np.uint32)

    def tokens(self, docs, n, unit, kind=0):
        text, off = _pack(docs)
        rc, st, tok_off, tok = self.raw(text, off, WORD if unit == "word" else CHAR, n, kind)
        assert rc == DSK_OK, self.lib.dsk_last_error()
        return st, tok_off, tok

    def sig(self, docs, n, unit, kind=0, num_perm=128):
        from datasketch_b200.shingle import signatures
        return signatures(docs, n, unit, num_perm=num_perm, hashfunc=HASHES[kind])


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def run(request):
    if request.param == "emu":
        return _Emu(request.getfixturevalue("emu_lib"))
    return _Gpu()


def _assert_tokens(run, docs, n, unit, kind=0):
    st, tok_off, tok = run.tokens(docs, n, unit, kind)
    bad, w_off, w_tok = _want(docs, n, unit, kind)
    assert np.array_equal(st[:-1] != 0, bad)
    assert st[-1] == (INVALID_UTF8 if bad.any() else 0)
    assert np.array_equal(tok_off, w_off)
    assert np.array_equal(tok, w_tok)


# ---- 1. the reference fixture ----------------------------------------------------------------------------------------
def test_shingles_equal_the_fixture(golden):
    g, docs = _fixture_docs(golden)
    for unit, n in CONFIGS:
        key = "%s%d" % (unit, n)
        flat, so, dp = _fixture_shingles(g, key)
        for i, d in enumerate(docs):
            want = [flat[so[j]:so[j + 1]] for j in range(dp[i], dp[i + 1])]
            assert shingles(d, n, unit) == want, (key, i)
            assert shingles(d.decode("utf-8"), n, unit) == want, (key, i)


def test_fixture_signatures(run, golden):
    """The tokens of all 320 documents are sha1_hash32 of the fixture's shingles; the signatures of the first 64 (those
    the fixture keeps) are the reference's MinHash.bulk."""
    g, docs = _fixture_docs(golden)
    for unit, n in CONFIGS:
        key = "%s%d" % (unit, n)
        flat, so, dp = _fixture_shingles(g, key)
        st, tok_off, tok = run.tokens(docs, n, unit)
        assert not st.any() and np.array_equal(tok_off, dp), key
        assert np.array_equal(tok, np.array([sha1_hash32(flat[so[j]:so[j + 1]]) for j in range(len(so) - 1)],
                                            dtype=np.uint32)), key
        want = g[key + "_sig"].astype(np.uint64)
        assert np.array_equal(run.sig(docs[:len(want)], n, unit), want), key


# ---- 2. hash kinds and K ---------------------------------------------------------------------------------------------
def test_hash_kinds_and_num_perm(run, golden):
    _, docs = _fixture_docs(golden)
    docs = docs[:120] if run.name == "emu" else docs
    for kind in (1, 2):
        for unit, n in (("word", 2), ("char", 3)):
            _assert_tokens(run, docs, n, unit, kind)
            if run.name != "gpu":
                continue
            import datasketch_b200 as dsk
            for k in (1, 64, 200, 256):
                want = np.stack([m.hashvalues for m in dsk.MinHash.bulk([shingles(d, n, unit) for d in docs],
                                                                        num_perm=k, hashfunc=HASHES[kind])])
                assert np.array_equal(run.sig(docs, n, unit, kind, num_perm=k), want), (kind, unit, n, k)


# ---- 3. whitespace ---------------------------------------------------------------------------------------------------
def test_whitespace_separators(run):
    if run.name == "gpu":
        cps = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    else:
        rs = np.random.RandomState(3)
        near = {c + d for c in WHITESPACE for d in (-1, 0, 1)} | {0x200B, 0x180E, 0xFEFF, 0x0, 0x7F, 0x80, 0x84, 0x86,
                                                                  0x9F, 0xA1, 0x167F, 0x1681, 0x2FFF, 0x3001}
        cps = sorted(near | set(int(c) for c in rs.randint(0, 0x110000, 300) if not 0xD800 <= c <= 0xDFFF))
    docs = [("a" + chr(c) + "b").encode("utf-8") for c in cps]
    for n in (1, 2):
        _assert_tokens(run, docs, n, "word")


# ---- 4. UTF-8 verdicts -----------------------------------------------------------------------------------------------
def _verdict_docs(run):
    rs = np.random.RandomState(4)
    if run.name == "gpu":
        docs = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
        docs += [bytes([a, b, c]) for a in range(0xE0, 0xF0) for b in range(256) for c in range(256)]
        four = rs.randint(0, 256, size=(200000, 4)).astype(np.uint8)
        four[:100000, 0] = rs.randint(0xF0, 0xF8, 100000)
        four[:50000, 1:] = rs.randint(0x80, 0xC0, (50000, 3))
        docs += [r.tobytes() for r in four]
        n_rand = 100000
    else:
        docs = [b"\x80", b"\xbf", b"\xc0\x80", b"\xc1\xbf", b"\xc2", b"\xc2\x7f", b"\xc2\xc0", b"\xe0\x80\x80",
                b"\xe0\x9f\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xee\x80\x80",
                b"\xef\xbf\xbf", b"\xe1\x80", b"\xf0\x8f\xbf\xbf", b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf",
                b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8\x88\x80\x80\x80", b"\xff", b"\xfe", b"a\x80b",
                b"\xc3\xa9\xa9", b"\xf0\x9f\x98", b"\xf0\x9f\x98\x80", b"ab\xe2\x82", b"\x00", b"\x7f", b""]
        docs += [bytes([a, b]) for a, b in rs.randint(0x7E, 0x100, (200, 2))]
        n_rand = 200
    lens = rs.randint(1, 13, n_rand)
    docs += [rs.randint(0x7E, 0x100, L).astype(np.uint8).tobytes() for L in lens]
    for ch in ("é", "中", "\U0001F600", "　"):      # a valid sequence split across two documents
        e = ch.encode("utf-8")
        for cut in range(1, len(e)):
            docs += [b"x" + e[:cut], e[cut:] + b"y"]
    return docs


def test_utf8_verdicts(run):
    docs = _verdict_docs(run)
    text, off = _pack(docs)
    rc, st, tok_off, _ = run.raw(text, off, CHAR, 1)
    assert rc == DSK_OK
    bad = []
    for d in docs:
        try:
            d.decode("utf-8")
            bad.append(False)
        except UnicodeDecodeError:
            bad.append(True)
    bad = np.array(bad)
    assert np.array_equal(st[:-1] != 0, bad)
    assert st[-1] == INVALID_UTF8
    assert np.array_equal(np.diff(tok_off)[bad], np.zeros(bad.sum(), dtype=np.int64))   # no shingles from a bad document


@pytest.mark.gpu
def test_api_raises_the_first_bad_documents_error():
    import torch
    from datasketch_b200.shingle import signatures
    docs = [b"fine", "café".encode(), b"ab\xed\xa0\x80cd", b"\xff", b"ok"]
    with pytest.raises(UnicodeDecodeError) as got:
        signatures(docs, 2, "char")
    with pytest.raises(UnicodeDecodeError) as want:
        docs[2].decode("utf-8")
    assert str(got.value) == str(want.value) and got.value.start == want.value.start
    assert got.value.object == want.value.object
    text, off = _pack(docs)
    with pytest.raises(UnicodeDecodeError) as got:
        signatures((torch.from_numpy(text.copy()).cuda(), torch.from_numpy(off).cuda()), 1, "word")
    assert str(got.value) == str(want.value)


# ---- 5. long and skewed ----------------------------------------------------------------------------------------------
def _words(rs, count):
    vocab = ["w%d" % i for i in range(500)] + ["é%d" % i for i in range(50)] + ["中文", "\U0001F600x"]
    seps = [" ", " ", " ", "\n", "\t ", "　", "  "]
    idx = rs.randint(0, len(vocab), count)
    sp = rs.randint(0, len(seps), count)
    return "".join(vocab[i] + seps[j] for i, j in zip(idx, sp))


def test_long_and_skewed(run):
    rs = np.random.RandomState(5)
    gpu = run.name == "gpu"
    small = [_words(rs, rs.randint(0, 30)).encode() for _ in range(50 if gpu else 12)]
    big = _words(rs, 1_500_000 if gpu else 6000).encode()
    word = (b"x" * (1 << 20)) if gpu else (b"y" * 20000)
    docs = small[:6] + [big] + small[6:] + [b" " + word + b" " + word[:1000] + b" a", "é".encode() * 3000]
    for unit, n in (("word", 1), ("word", 3)):
        _assert_tokens(run, docs, n, unit)
    chars = ["é中a\U0001F600 "[i % 5] for i in range(3000 if gpu else 600)]
    cdocs = ["".join(chars).encode(), b"short", "".join(chars[:999]).encode()]
    _assert_tokens(run, cdocs, 1000 if gpu else 200, "char")
    if gpu:   # through the signature kernel's piece path (documents longer than 4096 tokens)
        import datasketch_b200 as dsk
        want = np.stack([m.hashvalues for m in dsk.MinHash.bulk([shingles(d, 3, "word") for d in docs])])
        assert np.array_equal(run.sig(docs, 3, "word"), want)


# ---- 6. beyond 32-bit offsets ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_offsets_beyond_4gib():
    import torch
    from datasketch_b200.shingle import signatures
    rs = np.random.RandomState(6)
    docs = [_words(rs, rs.randint(1, 400)).encode() for _ in range(20)] + [b"", "中文 é".encode() * 50]
    base = (1 << 32) + 12345
    text, off = _pack(docs)
    big = torch.full((base + len(text) + 777,), 0x20, dtype=torch.uint8, device="cuda")
    big[base:base + len(text)] = torch.from_numpy(text.copy()).cuda()
    big[17:19] = torch.tensor([0x61, 0x62], dtype=torch.uint8)       # a word in the first (4 GiB) document
    # word bigrams: a first document of 4 GiB, whitespace but for one word; char 5-grams: nothing before the documents
    d_off = torch.from_numpy(np.concatenate([[0], base + off])).cuda()
    got = signatures((big, d_off), 2, "word")
    assert np.array_equal(got[1:], signatures(docs, 2, "word"))
    assert np.array_equal(got[0], signatures([b"ab"], 2, "word")[0])
    got = signatures((big, torch.from_numpy(base + off).cuda()), 5, "char")
    assert np.array_equal(got, signatures(docs, 5, "char"))
    del big


# ---- 7. device-resident flow -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpulsh_from_device_signatures():
    import datasketch_b200 as dsk
    from datasketch_b200.shingle import signatures
    rs = np.random.RandomState(7)
    base = [_words(rs, 200) for _ in range(300)]
    docs = base + [b[: len(b) * 9 // 10] + " extra words here" for b in base[:150]]
    host = signatures(docs, 3, "word")
    dev = signatures(docs, 3, "word", to_host=False)
    assert np.array_equal(dev.cpu().numpy().view(np.uint32), host.astype(np.uint32))
    a, b = dsk.GpuLSH(threshold=0.5, num_perm=128), dsk.GpuLSH(threshold=0.5, num_perm=128)
    a.insert(host[:300].astype(np.uint32))
    b.insert(dev[:300])
    def triples(res):
        ptr, idx, eq = (np.asarray(x) for x in res)
        return {(q, int(idx[i]), int(eq[i])) for q in range(len(ptr) - 1) for i in range(ptr[q], ptr[q + 1])}

    got = triples(b.query_jaccard(dev[300:], min_jaccard=0.5))
    assert got == triples(a.query_jaccard(host[300:].astype(np.uint32), min_jaccard=0.5))
    assert len({q for q, _, _ in got}) > 100     # most shortened copies find their original


@pytest.mark.gpu
def test_bulk_text_equals_bulk_over_shingles(golden):
    import datasketch_b200 as dsk
    _, docs = _fixture_docs(golden)
    texts = [d.decode("utf-8") for d in docs]
    for unit, n, kw in (("word", 2, {}), ("char", 3, {"num_perm": 64, "seed": 9, "hashfunc": murmur3_hash32})):
        got = dsk.MinHash.bulk_text(texts, n, unit, **kw)
        want = dsk.MinHash.bulk([shingles(t, n, unit) for t in texts], **kw)
        assert got == want
        assert all(g.seed == w.seed and len(g) == len(w) and g.hashfunc is w.hashfunc for g, w in zip(got, want))


# ---- 8. errors -------------------------------------------------------------------------------------------------------
def test_argument_errors_before_any_device_work():
    from datasketch_b200.hashfunc import sha1_hash64
    from datasketch_b200.shingle import signatures
    for n in (0, -1, 1.5, True, "2"):
        with pytest.raises(ValueError):
            signatures(["a b"], n=n)
    with pytest.raises(ValueError):
        signatures(["a b"], unit="byte")
    for hf in (sha1_hash64, lambda b: 1, hash):
        with pytest.raises(ValueError, match="MinHash.bulk"):
            signatures(["a b"], hashfunc=hf)


def test_c_abi_rejects_bad_arguments_and_offsets(run):
    lib = run.lib
    text, off = _pack([b"one two", b"three"])
    for unit, n in ((2, 1), (-1, 1), (WORD, 0), (CHAR, -3)):
        rc, *_ = run.raw(text, off, unit, n)
        assert rc == DSK_ERR_INVALID
    assert lib.dsk_shingle_count(None, None, 2, 0, WORD, 1, None, None, None, 0, None) == DSK_ERR_INVALID
    assert lib.dsk_shingle_hash(None, None, 2, 0, WORD, 1, 0, 0, None, None, None, 0, None) == DSK_ERR_INVALID
    st, tok_off, _ = run.tokens([b"a"], 1, "word")
    # a hash kind the library does not have
    if run.name == "emu":
        _keep, wsp, nb = run._ws(2, len(text))
        t_off = np.zeros(3, np.int64)
        out = np.zeros(4, np.uint32)
        assert lib.dsk_shingle_hash(text.ctypes.data, off.ctypes.data, 2, len(text), WORD, 1, 3, 0, t_off.ctypes.data,
                                    out.ctypes.data, wsp, nb, None) == DSK_ERR_INVALID
        assert lib.dsk_shingle_count(text.ctypes.data, off.ctypes.data, 2, len(text), WORD, 1, t_off.ctypes.data,
                                     out.ctypes.data, wsp, nb - 8, None) == DSK_ERR_INVALID
    # offsets that decrease or leave the text: flagged on the device, no shingles, nothing read through them
    for bad in ([0, 9, 5], [0, 5, len(text) + 1], [-1, 3, 5], [0, 1 << 40, len(text)]):
        rc, st, tok_off, tok = run.raw(text, np.array(bad, np.int64), WORD, 2)
        assert rc == DSK_OK and st[-1] & BAD_OFFSETS and not tok_off.any() and len(tok) == 0, bad


@pytest.mark.gpu
def test_api_errors():
    import torch
    from datasketch_b200.shingle import signatures
    for item in (3, None, ["a"], ("a", "b")):
        with pytest.raises(TypeError):
            signatures(["ok", item])
    with pytest.raises(UnicodeEncodeError):
        signatures(["ok", "lone \ud800 surrogate"])
    text = torch.from_numpy(np.frombuffer(b"one two three", np.uint8).copy()).cuda()
    for bad in ([0, 9, 5], [0, 5, 14], [-2, 3]):
        with pytest.raises(ValueError, match="offsets"):
            signatures((text, torch.tensor(bad, dtype=torch.int64, device="cuda")))
    with pytest.raises(ValueError):
        signatures((text, torch.tensor([0, 5], dtype=torch.int32, device="cuda")))
    assert signatures([]).shape == (0, 128)
    # bytes-like items of every kind, and str, give the same rows
    a = signatures(["héllo wörld", b"h\xc3\xa9llo", bytearray(b"x y"), memoryview(b"p q r")], 2)
    b = signatures([b"h\xc3\xa9llo w\xc3\xb6rld", "héllo", "x y", "p q r"], 2)
    assert np.array_equal(a, b)
