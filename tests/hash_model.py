"""Host model of the library's own hashes, and the adversarial inputs built from it (test infrastructure).

* ``band_fp`` / ``lsh_mix64`` (csrc/dsk_common.cuh): the 64-bit bucket fingerprint of an LSH band's r-tuple and the
  mix that picks its home slot in the band's open-addressed table.
* ``topk_fp16`` (csrc/jaccard_kernels.cu, fp_planes_kernel): the 16-bit value fingerprint of the top-k prefilter.

These are the library's hashes, not the reference's (the reference buckets by the tuple itself), so they live with the
tests rather than in oracle/.  The tests pin this model to the kernels bit for bit before they use it.

band_fp is  h = SEED ^ band;  h = (h ^ v) * MUL + ADD  for each of the r values;  fp = mix(h), with the table's empty
key remapped to EMPTY_KEY - 1.  Every step is a bijection of h (xor with v, multiplication by an odd constant,
addition), so two r-tuples collide exactly when they reach the same state h (or when one state mixes to EMPTY_KEY and
the other to EMPTY_KEY - 1).  For r = 1 the map from the value to the state is injective, so single values never
collide; r = 1 is only used to place tuples in chosen slots.  For r >= 2 a collision in the last two positions is a
32-bit condition on a free 32-bit value, which a meet-in-the-middle search over two 16-bit halves solves
(``_last_two``).
"""
import numpy as np

M64 = (1 << 64) - 1
SEED = 0x9E3779B97F4A7C15
MUL = 0xFF51AFD7ED558CCD
ADD = 0x2545F4914F6CDD1D
MIX = 0xD6E8FEB86659FD93
EMPTY_KEY = M64
MUL_INV = pow(MUL, -1, 1 << 64)
MIX_INV = pow(MIX, -1, 1 << 64)

_U = np.uint64


# ---- the hashes ---------------------------------------------------------------------------------------------------
def lsh_mix64(h):
    """lsh_mix64 of a uint64 array (or int)."""
    h = np.asarray(h, dtype=np.uint64)
    with np.errstate(over="ignore"):
        h = h ^ (h >> _U(32))
        h = h * _U(MIX)
        h = h ^ (h >> _U(32))
        h = h * _U(MIX)
        h = h ^ (h >> _U(32))
    return h


def tuple_states(tuples, band):
    """State of band_fp's multiply chain after every value of each row of ``tuples`` ([N, r] uint32), before the mix."""
    tuples = np.asarray(tuples, dtype=np.uint32)
    band = np.asarray(band, dtype=np.uint64)
    h = np.broadcast_to(_U(SEED) ^ band, tuples.shape[:1]).astype(np.uint64)
    with np.errstate(over="ignore"):
        for q in range(tuples.shape[1]):
            h = (h ^ tuples[:, q].astype(np.uint64)) * _U(MUL) + _U(ADD)
    return h


def _remap(fp):
    return np.where(fp == _U(EMPTY_KEY), _U(EMPTY_KEY - 1), fp)


def tuple_fp(tuples, band):
    """band_fp of each row of ``tuples`` ([N, r]) as band ``band`` (an int or an [N] array)."""
    return _remap(lsh_mix64(tuple_states(tuples, band)))


def band_fp(sig, b, r):
    """[N, K] uint32 signatures -> [N, b] uint64 bucket fingerprints (what dsk_band_fingerprints returns)."""
    sig = np.asarray(sig, dtype=np.uint32)
    return np.stack([tuple_fp(sig[:, j * r:(j + 1) * r], j) for j in range(b)], axis=1)


def cap_slots(capacity):
    """Slots per band table of an index created for ``capacity`` documents (dsk_lsh_create)."""
    s = 1024
    while s < 2 * capacity:
        s <<= 1
    return s


def home_slot(fp, capacity):
    return lsh_mix64(fp) & _U(cap_slots(capacity) - 1)


def topk_fp16(v):
    """The prefilter's 16-bit fingerprint of each uint32 value."""
    v = np.asarray(v, dtype=np.uint32)
    return (v ^ (v >> np.uint32(16))) & np.uint32(0xFFFF)


def fp16_twins(v, rng):
    """Values with the same 16-bit fingerprint as ``v`` but different from it: v ^ (x * 0x00010001), x in 1..0xFFFF."""
    v = np.asarray(v, dtype=np.uint32)
    x = rng.randint(1, 1 << 16, size=v.shape).astype(np.uint32)
    return v ^ (x * np.uint32(0x00010001))


# ---- preimages -----------------------------------------------------------------------------------------------------
def _step(h, v):
    return ((h ^ v) * MUL + ADD) & M64


def _state(values, band):
    h = SEED ^ band
    for v in values:
        h = _step(h, int(v))
    return h


def mix_inverse(fp):
    """The state h with lsh_mix64(h) == fp (python ints)."""
    h = fp ^ (fp >> 32)
    h = (h * MIX_INV) & M64
    h ^= h >> 32
    h = (h * MIX_INV) & M64
    return h ^ (h >> 32)


_HALF = np.arange(1 << 16, dtype=np.uint64)


def _last_two(hp, target):
    """Every (a, b) of 32-bit values with _step(_step(hp, a), b) == target.

    _step(h1, b) == target  <=>  h1 ^ b == T := (target - ADD) * MUL^-1, so h1 = _step(hp, a) must have the high word of
    T.  With xl = low32(hp) ^ a (free), h1 = xl * MUL + D (mod 2^64), D = high32(hp) * 2^32 * MUL + ADD; xl = xh * 2^16 +
    xlo splits h1 into A[xh] + B[xlo], whose high words add up to high32(T) (with or without a carry from the low
    words).  Sort one side, binary-search the other, verify each hit exactly."""
    T = ((target - ADD) * MUL_INV) & M64
    t_hi = T >> 32
    D = (((hp >> 32) << 32) * MUL + ADD) & M64
    with np.errstate(over="ignore"):
        A = _HALF * _U((MUL << 16) & M64)
        B = _HALF * _U(MUL) + _U(D)
        hi_a, hi_b = A >> _U(32), B >> _U(32)
        order = np.argsort(hi_a, kind="stable")
        sa = hi_a[order]
        out = set()
        for carry in (0, 1):
            need = (_U(t_hi) - hi_b - _U(carry)) & _U(0xFFFFFFFF)
            lo, hi = np.searchsorted(sa, need, "left"), np.searchsorted(sa, need, "right")
            for xlo in np.nonzero(hi > lo)[0]:
                for j in range(lo[xlo], hi[xlo]):
                    xl = (int(order[j]) << 16) | int(xlo)
                    h1 = ((((hp >> 32) << 32) | xl) * MUL + ADD) & M64
                    if h1 >> 32 == t_hi:
                        out.add((xl ^ (hp & 0xFFFFFFFF), (h1 ^ T) & 0xFFFFFFFF))
    return sorted(out)


def tuple_with_state(state, band, r, rng, tries=64):
    """An r-tuple (r >= 2) whose band_fp chain reaches ``state`` as band ``band``, or None.  For r == 2 there is one
    candidate prefix (the band's seed), so it may not exist; for r > 2 random prefixes are tried."""
    assert r >= 2
    for _ in range(tries if r > 2 else 1):
        prefix = [int(x) for x in rng.randint(0, 1 << 32, size=r - 2, dtype=np.uint64)]
        sols = _last_two(_state(prefix, band), state)
        if sols:
            return np.array(prefix + list(sols[0]), dtype=np.uint32)
    return None


def tuple_with_prefp(fp, band, r, rng, tries=64):
    """An r-tuple whose fingerprint BEFORE the empty-key remap is ``fp`` (e.g. EMPTY_KEY itself), or None."""
    return tuple_with_state(mix_inverse(fp), band, r, rng, tries)


def second_preimage(tup, band, rng, avoid=(), tries=64):
    """An r-tuple (r >= 2) different from ``tup`` and from every tuple in ``avoid``, with the same band_fp as band
    ``band``, or None.  The last two values are solved for; when the original prefix has no further solution (r > 2),
    the third value from the end is redrawn."""
    tup = [int(x) for x in tup]
    seen = {tuple(tup)} | {tuple(int(x) for x in t) for t in avoid}
    r = len(tup)
    assert r >= 2
    target = _state(tup, band)
    prefix = tup[:-2]
    for t in range(tries if r > 2 else 1):
        if t > 0:
            prefix[-1] = int(rng.randint(0, 1 << 32, dtype=np.uint64))
        for a, b in _last_two(_state(prefix, band), target):
            cand = prefix + [a, b]
            if tuple(cand) not in seen:
                return np.array(cand, dtype=np.uint32)
    return None
