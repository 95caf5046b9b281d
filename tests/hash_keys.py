"""Keys built to collide in the hash tables of the Grouper (csrc/grouper.cu), the fused group-by (csrc/groupby_fused.cu,
groupby_partitioned.cuh) and everything built on them.

hash64 (murmur3 fmix64, hash_table.cuh) is a bijection on 64-bit words, and for one 8-byte key column the encoded key IS
the raw bits.  So a test picks the hash values it wants -- equal low bits (one table home slot), equal bits 20.. (one
pre-aggregation slot), equal radix digits (one partition) -- and inverts them to get the keys.  The constants the cases aim
at are read from the sources, so a retune keeps the cases on target."""
import os
import re

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_b200", "csrc")
M64 = (1 << 64) - 1
_C1, _C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
_C1_INV, _C2_INV = pow(_C1, -1, 1 << 64), pow(_C2, -1, 1 << 64)


# ---- fmix64 and its inverse, on Python ints and on uint64 arrays ---------------------------------------------------
def fmix64(k: int) -> int:
    k &= M64
    k ^= k >> 33
    k = (k * _C1) & M64
    k ^= k >> 33
    k = (k * _C2) & M64
    k ^= k >> 33
    return k


def fmix64_inverse(h: int) -> int:
    # x ^= x >> 33 is its own inverse on 64 bits (a second shift by 33 leaves nothing)
    h &= M64
    h ^= h >> 33
    h = (h * _C2_INV) & M64
    h ^= h >> 33
    h = (h * _C1_INV) & M64
    h ^= h >> 33
    return h


def fmix64_np(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k).astype(np.uint64)
    with np.errstate(over="ignore"):
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(_C1)
        k = k ^ (k >> np.uint64(33))
        k = k * np.uint64(_C2)
        k = k ^ (k >> np.uint64(33))
    return k


def fmix64_inverse_np(h: np.ndarray) -> np.ndarray:
    h = np.asarray(h).astype(np.uint64)
    with np.errstate(over="ignore"):
        h = h ^ (h >> np.uint64(33))
        h = h * np.uint64(_C2_INV)
        h = h ^ (h >> np.uint64(33))
        h = h * np.uint64(_C1_INV)
        h = h ^ (h >> np.uint64(33))
    return h


# ---- constants, read from the sources --------------------------------------------------------------------------------
def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _int(text, pattern):
    m = re.search(pattern, text)
    assert m, pattern
    return int(m.group(1), 0)


def _shift(text, name):
    m = re.search(rf"constexpr \w+ {name} = 1ll? << (\d+);", text) or re.search(rf"constexpr \w+ {name} = 1ull << (\d+);", text)
    assert m, name
    return 1 << int(m.group(1))


_HT, _GR, _GP, _GF, _HJ = (_read(f) for f in ("hash_table.cuh", "grouper.cu", "groupby_partitioned.cuh",
                                              "groupby_fused.cu", "hash_join.cu"))
MAX_PROBE = _int(_HT, r"constexpr int kMaxProbe = (\d+);")
EMPTY_KEY = _int(_HT, r"constexpr uint64_t kEmptyKey = (0x[0-9a-fA-F]+)ull;")
DIRECT_MAX_RANGE = _shift(_GR, "kDirectMaxRange")
PRE_SLOTS = _int(_GP, r"constexpr int kPreSlots = (\d+);")
PRE_PROBE = _int(_GP, r"constexpr int kPreProbe = (\d+);")
PART_RADIX = _int(_GP, r"constexpr int kPartRadix = (\d+);")
PART_MIN_ROWS = _shift(_GF, "kPartMinRows")
SCAN_TILE = _int(_HJ, r"constexpr int kScanTile = (\d+);")
# the Grouper's first table guess: next_pow2(n < SMALL ? FLOOR : (n < 1 << MID ? MUL * n : 1 << TOP))
_g = re.search(r"n < (\d+) \? (\d+) : \(n < \(1 << (\d+)\) \? (\d+) \* n : \(1 << (\d+)\)\)", _GR)
assert _g, "first-guess rule"
GUESS_SMALL, GUESS_FLOOR, GUESS_MID, GUESS_MUL, GUESS_TOP = (int(x) for x in _g.groups())
# direct-window eligibility of a first batch: width < max(ROOMY_MUL * n, ROOMY_MIN)
_r = re.search(r"roomy = \(uint64_t\)n \* (\d+) > (\d+)", _GR)
assert _r, "roomy rule"
ROOMY_MUL, ROOMY_MIN = int(_r.group(1)), int(_r.group(2))
# the direct table's size: next_pow2(max(2 * span, DIRECT_FLOOR)), at most kDirectMaxRange
DIRECT_FLOOR = _int(_GR, r"span \* 2 < (\d+) \? \d+ : span \* 2")
# the fused table's first size without expected_groups, and the smallest table the partitioned path starts from
FUSED_FIRST_CAP = 1 << _int(_GF, r"expected_groups \* 2 : \(1u << (\d+)\)\)")
FUSED_PART_CAP = 2 << _int(_GF, r"g->hint : \(1 << (\d+)\)\)\), s\)\);")


def next_pow2(v: int) -> int:
    r = 1
    while r < v:
        r <<= 1
    return r


# ---- key builders ---------------------------------------------------------------------------------------------------
def _fields_mask(fields):
    mask = val = 0
    for shift, nbits, value in fields:
        m = ((1 << nbits) - 1) << shift
        assert not (mask & m), "overlapping fields"
        mask |= m
        val |= (value << shift) & m
    return mask, val


def hashes_with_fields(n: int, fields, seed: int) -> np.ndarray:
    """n distinct 64-bit hash values that take `value` on bits [shift, shift + nbits) for every (shift, nbits, value) of
    `fields`; the other bits are random.  None of them inverts to the empty-marker key."""
    mask, val = _fields_mask(fields)
    free = 64 - bin(mask).count("1")
    assert free >= 1 and n <= (1 << free) - 1, "not enough free bits for n distinct keys"
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    forbidden = fmix64(EMPTY_KEY)
    while len(out) < n:
        r = int(rng.integers(0, 1 << 63, dtype=np.int64)) << 1 | int(rng.integers(0, 2))
        h = (r & ~mask & M64) | val
        if h in seen or h == forbidden:
            continue
        seen.add(h)
        out.append(h)
    return np.array(out, dtype=np.uint64)


def keys_with_fields(n: int, fields, seed: int, dtype=np.int64) -> np.ndarray:
    """n distinct keys of an 8-byte type (int64 / uint64 / float64, as raw bits) whose hash64 takes the given fields"""
    return fmix64_inverse_np(hashes_with_fields(n, fields, seed)).view(dtype)


def filler_keys(n: int, avoid, seed: int, dtype=np.int64, exclude=()) -> np.ndarray:
    """n distinct random keys whose hash64 matches NONE of the `avoid` field sets (each a list of fields), none equal to
    the empty marker or to a key of `exclude`"""
    rng = np.random.default_rng(seed)
    ex = set(np.asarray(exclude).view(np.uint64).tolist()) if len(exclude) else set()
    out, seen = [], set()
    while len(out) < n:
        cand = rng.integers(0, np.iinfo(np.int64).max, 2 * (n - len(out)) + 16, dtype=np.int64).view(np.uint64)
        cand = cand ^ (rng.integers(0, 2, len(cand)).astype(np.uint64) << np.uint64(63))
        h = fmix64_np(cand)
        ok = cand != np.uint64(EMPTY_KEY)
        for fields in avoid:
            mask, val = _fields_mask(fields)
            ok &= (h & np.uint64(mask)) != np.uint64(val)
        for c in cand[ok].tolist():
            if c not in seen and c not in ex:
                seen.add(c)
                out.append(c)
                if len(out) == n:
                    break
    return np.array(out, dtype=np.uint64).view(dtype)


def slot_field(bits: int, value: int = 0x5A5A5A5A5A5A5A5A):
    """hash & (2^bits - 1) fixed: one home slot in every table of up to 2^bits slots"""
    return [(0, bits, value)]


def pre_slot_field(value: int = 0x2A5):
    """(hash >> 20) & (kPreSlots - 1) fixed: one shared-memory pre-aggregation slot"""
    return [(20, PRE_SLOTS.bit_length() - 1, value)]


def consecutive_keys_with_low_bits(n: int, bits: int, start: int = 0, value: int = 0x1234567):
    """the first n integers >= start whose hash64 has the given low `bits`: a cluster of keys that also fits a
    direct-addressed window (about n * 2^bits wide)"""
    want = value & ((1 << bits) - 1)
    out, lo, step = [], start, max(1 << 20, n << bits)
    while len(out) < n:
        cand = np.arange(lo, lo + step, dtype=np.uint64)
        hit = cand[(fmix64_np(cand) & np.uint64((1 << bits) - 1)) == np.uint64(want)]
        out.extend(hit[: n - len(out)].tolist())
        lo += step
    return np.array(out, dtype=np.uint64).view(np.int64)
