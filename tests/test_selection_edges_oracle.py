"""Pins tests/selection_ref.py (the byte-exact Filter / Take reference of the GPU selection tests) against pyarrow.compute
on every value layout the device accepts: all integer widths, float16/32/64 with NaN payloads, -0.0 and the other special
bit patterns, the temporal types (carried as their int32 / int64 storage), fixed_size_binary of widths 1 to 17, bool, the
four string types and dictionaries with all eight index types.  Shapes: slice offsets, both null behaviours, empty values
with all-null indices, and the IndexError cases.

The int32-offset capacity rule is kept out of this comparison: the installed pyarrow predates the reference's Take check
(vector_selection_internal.cc:484,519-523) and silently wraps the last offset of a 2048 x 1 MiB take to -2^31.  The rule is
pinned to the source's numbers in test_capacity_rule_matches_the_source instead, and checked on the device by
test_gpu_selection_edges.py."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import exact_ref as er
from tests import selection_ref as sr
from tests.util import SEED, random_array

INDEX_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()]
STRING_TYPES = [pa.string(), pa.large_string(), pa.binary(), pa.large_binary()]
FIXED_LAYOUTS = INDEX_TYPES + [
    pa.float16(), pa.float32(), pa.float64(), pa.date32(), pa.time32("ms"), pa.time64("us"), pa.timestamp("us", tz="UTC"),
    pa.duration("ns"), pa.date64(),
] + [pa.binary(w) for w in (1, 2, 3, 4, 8, 12, 16, 17)]

# special bit patterns per byte width: the float16/32/64 NaNs with and without payload, signalling NaNs, -0.0, infinities,
# denormals and all-ones; wider rows repeat float64 patterns, the others hold sign-bit and all-ones bytes
F16_SPECIAL = [0x0000, 0x8000, 0x7E00, 0xFE00, 0x7E5A, 0x7C01, 0xFFFF, 0x7C00, 0xFC00, 0x0001]


def special_rows(w: int) -> np.ndarray:
    """(k, w) uint8 rows of special bit patterns for a w-byte layout"""
    if w == 2:
        pats = np.array(F16_SPECIAL, np.uint16)
    elif w == 4:
        pats = np.array(list(er.F32_SPECIAL.values()), np.uint32)
    elif w in (8, 16):
        pats = np.array(list(er.F64_SPECIAL.values()), np.uint64)
        if w == 16:
            pats = np.stack([pats, pats[::-1]], axis=1)
    else:
        return np.array([[b] * w for b in (0x00, 0x80, 0xFF, 0x7F)], np.uint8)
    return np.ascontiguousarray(pats).view(np.uint8).reshape(len(pats), w)


def in_range_bytes(t: pa.DataType, m: int, rng) -> np.ndarray:
    """random row bytes; time32 / time64 values are drawn within a day, which Arrow's full validation requires"""
    w = sr.byte_width(t)
    if pa.types.is_time32(t) or pa.types.is_time64(t):
        day = {"s": 86400, "ms": 86400 * 10**3, "us": 86400 * 10**6, "ns": 86400 * 10**9}[t.unit]
        v = rng.integers(0, day, m, dtype=np.int64).astype(np.int32 if w == 4 else np.int64)
        return v.view(np.uint8).reshape(m, w)
    b = rng.integers(0, 256, (m, w), dtype=np.uint8)
    if not pa.types.is_temporal(t):
        sp = special_rows(w)
        rows = np.arange(0, m, 7)
        b[rows] = sp[np.arange(len(rows)) % len(sp)]
    return b


def bitmap(valid: np.ndarray) -> pa.Buffer:
    return pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())


def fixed_array(t: pa.DataType, n: int, rng, null_p=0.1, offset=0, data: np.ndarray = None) -> pa.Array:
    """n rows of layout t (a slice at `offset` of a longer array); every 7th row holds a special bit pattern"""
    m = n + offset
    b = in_range_bytes(t, m, rng) if data is None else data
    valid = rng.random(m) >= null_p
    bufs = [bitmap(valid) if null_p > 0 else None, pa.py_buffer(np.ascontiguousarray(b).tobytes())]
    arr = pa.Array.from_buffers(t, m, bufs, null_count=-1 if null_p > 0 else 0)
    return arr.slice(offset) if offset else arr


def bool_array(n: int, rng, p_true=0.5, null_p=0.1, offset=0) -> pa.Array:
    m = n + offset
    arr = pa.array(rng.random(m) < p_true, pa.bool_(), mask=(rng.random(m) < null_p) if null_p > 0 else None)
    return arr.slice(offset) if offset else arr


def index_array(t: pa.DataType, n: int, n_values: int, rng, null_p=0.1, offset=0) -> pa.Array:
    """in-bounds indices of type t, with 0 and n_values - 1 at the first and last row"""
    hi = min(n_values - 1, np.iinfo(t.to_pandas_dtype()).max)
    m = n + offset
    v = rng.integers(0, hi, m, dtype=t.to_pandas_dtype(), endpoint=True)
    if n:
        v[offset], v[-1] = 0, hi
    arr = pa.array(v, t, mask=(rng.random(m) < null_p) if null_p > 0 else None)
    return arr.slice(offset) if offset else arr


def dictionary_array(index_type: pa.DataType, n: int, rng, null_p=0.1) -> pa.DictionaryArray:
    """a string dictionary with a null entry (index 1), so a valid index can point at a null value"""
    dictionary = pa.array(["a", None, "", "ccc", "dd"] + [f"v{i}" for i in range(60)])
    return pa.DictionaryArray.from_arrays(index_array(index_type, n, len(dictionary), rng, null_p), dictionary)


def check_filter(values, mask, msg=""):
    for ns in (sr.DROP, sr.EMIT_NULL):
        want = sr.filter(values, mask, ns)
        sr.assert_rows_equal(pc.filter(values, mask, null_selection_behavior=ns), want, f"{msg} {ns}")
        assert sr.filter_output_size(mask, ns) == len(want)


def check_take(values, indices, msg=""):
    sr.assert_rows_equal(pc.take(values, indices), sr.take(values, indices), msg)


@pytest.mark.parametrize("t", FIXED_LAYOUTS, ids=str)
def test_fixed_width_layouts(t):
    rng = np.random.default_rng(SEED)
    for n, off, moff in ((0, 0, 0), (1, 0, 0), (300, 0, 0), (300, 5, 3), (1000, 16, 13)):
        for null_p in (0.0, 0.2):
            v = fixed_array(t, n, rng, null_p, off)
            check_filter(v, bool_array(n, rng, 0.5, 0.1, moff), f"{t} n={n} off={off}")
            check_filter(v, bool_array(n, rng, 0.5, 0.0, moff), f"{t} n={n} off={off} mask non-null")
            for it in INDEX_TYPES:
                if n:
                    check_take(v, index_array(it, 257, n, rng, 0.1, 3), f"{t} {it} n={n}")


def test_bit_patterns_survive_byte_for_byte():
    """the reference keeps NaN payloads and -0.0 apart, and so does pyarrow: canonicalising them must fail the check"""
    for t in (pa.float16(), pa.float32(), pa.float64()):
        w = sr.byte_width(t)
        sp = special_rows(w)
        v = fixed_array(t, len(sp), np.random.default_rng(SEED), 0.0, data=sp)
        got = sr.filter(v, pa.array([True] * len(sp)))
        assert got.data.tobytes() == sp.tobytes()
        sr.assert_rows_equal(pc.take(v, pa.array(range(len(sp)), pa.int32())), sr.take(v, pa.array(range(len(sp)))))
        canon = sp.copy()
        canon[1] = sp[0]  # -0.0 -> +0.0
        with pytest.raises(AssertionError, match="rows differ"):
            sr.assert_rows_equal(fixed_array(t, len(sp), np.random.default_rng(SEED), 0.0, data=canon), got)


def test_bool():
    rng = np.random.default_rng(SEED + 1)
    for n, off, moff in ((1, 0, 0), (700, 0, 0), (700, 3, 5), (5000, 61, 7)):
        for null_p in (0.0, 0.3):
            v = bool_array(n, rng, 0.5, null_p, off)
            check_filter(v, bool_array(n, rng, 0.3, 0.2, moff), f"bool n={n}")
            for it in INDEX_TYPES:
                check_take(v, index_array(it, 200, n, rng, 0.2, 1), f"bool {it} n={n}")


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_strings(t):
    rng = np.random.default_rng(SEED + 2)
    for n, off, lo, hi in ((1, 0, 0, 5), (600, 0, 0, 32), (600, 3, 0, 3), (300, 7, 40, 90)):
        for null_p in (0.0, 0.2):
            v = random_array(t, n, null_p, SEED + n + off, lo=lo, hi=hi, offset=off)
            check_filter(v, bool_array(n, rng, 0.5, 0.2, 2), f"{t} n={n}")
            for it in INDEX_TYPES:
                check_take(v, index_array(it, 150, n, rng, 0.2, 2), f"{t} {it} n={n}")


@pytest.mark.parametrize("it", INDEX_TYPES, ids=str)
def test_dictionaries(it):
    rng = np.random.default_rng(SEED + 3)
    d = dictionary_array(it, 500, rng)
    assert (np.asarray(d.indices.to_numpy(zero_copy_only=False)) == 1).any(), "no valid index at the null entry"
    check_filter(d, bool_array(500, rng, 0.5, 0.1), str(it))
    check_filter(d.slice(9), bool_array(491, rng, 0.5, 0.1, 3), f"{it} sliced")
    for jt in (pa.int8(), pa.uint32(), pa.int64()):
        check_take(d, index_array(jt, 300, 500 if jt != pa.int8() else 128, rng, 0.1), f"{it} {jt}")


def test_empty_values_all_null_indices():
    for t in (pa.int32(), pa.binary(16), pa.bool_(), pa.string(), pa.large_binary()):
        empty = pa.array([], t)
        for it in (pa.int8(), pa.uint64()):
            idx = pa.array([None, None, None], it)
            got = sr.take(empty, idx)
            assert got.null_count() == 3
            sr.assert_rows_equal(pc.take(empty, idx), got, f"{t} {it}")
        assert len(sr.take(empty, pa.array([], pa.int32()))) == 0
        check_filter(empty, pa.array([], pa.bool_()), str(t))


def test_all_null_mask():
    v = fixed_array(pa.int64(), 100, np.random.default_rng(SEED), 0.1)
    mask = pa.array([None] * 100, pa.bool_())
    assert len(sr.filter(v, mask, sr.DROP)) == 0
    assert sr.filter(v, mask, sr.EMIT_NULL).null_count() == 100
    check_filter(v, mask)


BAD_INDEX_CASES = [  # (type, indices): the first VALID out-of-range row is reported
    (pa.int8(), [0, -1, 5, -128]),
    (pa.int8(), [None, 0, 127, -3]),
    (pa.uint8(), [2, 255, 0, 7]),
    (pa.int16(), [1, 2, -32768, 99]),
    (pa.uint16(), [65535, 3]),
    (pa.int32(), [4, -2147483648, 9]),
    (pa.uint32(), [0, 4294967295]),
    (pa.int64(), [0, 1, -1, 10]),
    (pa.int64(), [9223372036854775807]),
    (pa.uint64(), [0, 9223372036854775813, 6]),
    (pa.uint64(), [18446744073709551615]),
]


@pytest.mark.parametrize("t,idx", BAD_INDEX_CASES, ids=lambda x: str(x))
def test_index_errors(t, idx):
    for values in (pa.array(list(range(5)), pa.int32()), pa.array(["a", "b", None, "d", "e"]),
                   pa.array([True, False, None, True, True])):
        i = pa.array(idx, t)
        with pytest.raises(pa.ArrowIndexError) as want:
            pc.take(values, i)
        with pytest.raises(pa.ArrowIndexError) as got:
            sr.take(values, i)
        assert str(got.value) == str(want.value)


def test_bad_index_under_a_null_is_not_checked():
    values = pa.array([10, 20, 30], pa.int16())
    idx = pa.Array.from_buffers(pa.int32(), 3, [bitmap(np.array([True, False, True])),
                                                pa.py_buffer(np.array([2, 1000, 0], np.int32).tobytes())], null_count=1)
    got = sr.take(values, idx)
    sr.assert_rows_equal(pc.take(values, idx), got)
    assert got.valid.tolist() == [True, False, True]


@pytest.mark.parametrize("n", [1, 5000, 65535, 65536, 70001])
def test_take_indices(n):
    rng = np.random.default_rng(SEED + n)
    mask = bool_array(n, rng, 0.3, 0.2, 3)
    for ns in (sr.DROP, sr.EMIT_NULL):
        got = sr.take_indices(mask, ns)
        assert got.type == (pa.uint16() if n <= 65535 else pa.uint32())
        want = pc.filter(pa.array(np.arange(n), got.type), mask, null_selection_behavior=ns)
        sr.assert_rows_equal(want, got, f"{n} {ns}")


def test_capacity_rule_matches_the_source():
    """kOffsetLimit = INT32_MAX - 1, checked against the running total before each append (Take only)"""
    mib = 1 << 20
    assert not sr.take_overflows([mib] * 2047 + [mib - 2])  # total 2^31 - 2
    assert sr.take_overflows([mib] * 2047 + [mib - 1])      # total 2^31 - 1
    assert not sr.take_overflows([mib] * 2047)
    assert sr.take_overflows([mib] * 2048)                  # the reference's TakeBinaryOffsetOverflow
    assert not sr.filter_overflows([mib] * 2047 + [mib - 1])
    # through take(): the sizes of VALID taken rows count, a null row adds nothing
    values = pa.array([b"x" * 3, b"y"], pa.binary())
    idx = pa.array([0, None, 1], pa.int32())
    assert sr.take(values, idx).data[0] == b"xxx"
