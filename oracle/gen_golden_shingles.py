"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/shingles.npz: word and character n-gram shingles of a seeded text
corpus and the REAL reference's MinHash.bulk signatures of them.

Run where an ekzhu/datasketch checkout exists (it imports the reference from it):

    DATASKETCH_REF=<ekzhu/datasketch checkout> python oracle/gen_golden_shingles.py

The reference has no shingling code; it leaves it to the user.  The definition below is this generator's own statement
of datasketch_b200/shingle.py:shingles() (words are str.split(), joined by one space; characters are code points; a
document shorter than n gives one shingle of all its units, an empty one none).  The corpus (320 documents) mixes ASCII
prose, 2-, 3- and 4-byte characters, combining marks, every one of Python's 29 whitespace code points as separators (in
runs and at both ends), U+200B / U+180E / U+FEFF, NUL, empty and whitespace-only documents and documents shorter than n.
Stored: the UTF-8 corpus (bytes + offsets); for word n in {1, 3, 5} and char n in {1, 4, 9}, the shingles (their bytes
back to back, the length of each as uint16, the number per document as int32); and, for the first N_SIG = 64 documents
(the 17 written out by hand and 47 seeded ones), datasketch.MinHash.bulk at num_perm = 128, seed 1, sha1_hash32 (stored
as uint32: every value fits 32 bits).  Signatures are random 32-bit values that do not compress, so they are kept for a
prefix only; the shingle lists of all 320 documents pin the tokens.
"""
from __future__ import annotations

import os
import sys

import numpy as np

REF = os.environ["DATASKETCH_REF"]
sys.path.insert(0, REF)
from datasketch import MinHash  # noqa: E402  (the reference)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
WHITESPACE = [0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x1C, 0x1D, 0x1E, 0x1F, 0x20, 0x85, 0xA0, 0x1680] + \
    list(range(0x2000, 0x200B)) + [0x2028, 0x2029, 0x202F, 0x205F, 0x3000]
CONFIGS = [("word", 1), ("word", 3), ("word", 5), ("char", 1), ("char", 4), ("char", 9)]
N_SIG = 64


def definition(text: str, n: int, unit: str):
    units = text.split() if unit == "word" else list(text)
    sep = " " if unit == "word" else ""
    m = len(units)
    if m == 0:
        return []
    if m < n:
        return [sep.join(units).encode("utf-8")]
    return [sep.join(units[i:i + n]).encode("utf-8") for i in range(m - n + 1)]


def corpus(rs):
    assert len(WHITESPACE) == 29 and all(chr(c).isspace() for c in WHITESPACE)
    prose = ("the quick brown fox jumps over the lazy dog while seven wizards quietly judge boxing matches near "
             "an old harbour").split()
    other = ["café", "naïve", "Straße", "日本語", "中文", "한국어", "Ελληνικά", "русский", "עברית", "عربي",
             "\U0001F600", "\U0001F9EA\U0001F52C", "𝔘𝔫𝔦𝔠𝔬𝔡𝔢", "é", "ạ̈", "​", "᠎", "﻿",
             "x​y", "nul\x00byte", "\x00"]
    docs = ["", " ", "\t\n", "".join(chr(c) for c in WHITESPACE), "a", "ab", "a b", "日", "\U0001F600", "\x00",
            "​", "᠎﻿", "one two", "one two three four", " lead", "trail ", chr(0x3000) + "x" + chr(0x85)]
    while len(docs) < 320:
        words = []
        for _ in range(rs.randint(0, 40)):
            words.append(prose[rs.randint(len(prose))] if rs.rand() < 0.7 else other[rs.randint(len(other))])
        seps = []
        for _ in range(len(words) + 1):
            r = rs.rand()
            if r < 0.6:
                seps.append(" ")
            else:
                seps.append("".join(chr(WHITESPACE[rs.randint(29)]) for _ in range(rs.randint(1, 4))))
        text = seps[0] if rs.rand() < 0.3 else ""
        for i, w in enumerate(words):
            text += w + (seps[i + 1] if i + 1 < len(words) or rs.rand() < 0.3 else "")
        docs.append(text)
    return docs


def main():
    rs = np.random.RandomState(20261018)
    docs = corpus(rs)
    enc = [d.encode("utf-8") for d in docs]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(e) for e in enc], out=off[1:])
    out = {"text": np.frombuffer(b"".join(enc), dtype=np.uint8), "offsets": off}
    for unit, n in CONFIGS:
        sh = [definition(d, n, unit) for d in docs]
        flat = [s for d in sh for s in d]
        lens = np.array([len(s) for s in flat], dtype=np.int64)
        assert lens.max() < 1 << 16
        sig = np.stack([m.hashvalues for m in MinHash.bulk(sh[:N_SIG], num_perm=128)])
        assert sig.max() < 1 << 32   # stored as uint32 (values of sha1_hash32 tokens fit 32 bits)
        key = "%s%d" % (unit, n)
        out[key + "_bytes"] = np.frombuffer(b"".join(flat), dtype=np.uint8)
        out[key + "_len"] = lens.astype(np.uint16)
        out[key + "_count"] = np.array([len(d) for d in sh], dtype=np.int32)
        out[key + "_sig"] = sig.astype(np.uint32)
    np.savez_compressed(os.path.join(OUT, "shingles.npz"), **out)
    print("wrote shingles.npz:", len(docs), "documents,", len(out["text"]), "bytes")


if __name__ == "__main__":
    main()
