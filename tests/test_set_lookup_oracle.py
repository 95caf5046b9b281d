"""The host restatement of is_in / index_in (set_lookup_ref) against pyarrow.compute (MATCH and SKIP, the behaviours
pyarrow's Python exposes) and against the reference's own expected outputs (tests/golden/kat_set_lookup.json, all four
behaviours).  CPU only."""
import json
import os
import struct
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import set_lookup_ref as ref

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_set_lookup.json")))
TYPES = {"bool": pa.bool_(), "int8": pa.int8(), "uint8": pa.uint8(), "int16": pa.int16(), "uint16": pa.uint16(),
         "int32": pa.int32(), "uint32": pa.uint32(), "int64": pa.int64(), "uint64": pa.uint64(), "float": pa.float32(),
         "double": pa.float64(), "string": pa.string(), "binary": pa.binary(), "large_string": pa.large_string(),
         "large_binary": pa.large_binary()}
NUMERIC = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float", "double"]
STRINGS = ["string", "binary", "large_string", "large_binary"]


def _py(v, t):
    if v is not None and t in (pa.binary(), pa.large_binary()):
        return v.encode()
    return v


def _arr(values, t):
    return pa.array([_py(v, t) for v in values], t)


@pytest.mark.parametrize("case", range(len(KAT["cases"])))
def test_kat(case):
    c = KAT["cases"][case]
    for tname in c["types"]:
        t = TYPES[tname]
        got = ref.expected(_arr(c["values"], t), _arr(c["value_set"], t), c["behavior"], c["function"])
        want = pa.array(c["expected"], pa.int32() if c["function"] == "index_in" else pa.bool_())
        assert got.equals(want), (c, tname, got)


@pytest.mark.parametrize("case", range(len(KAT["casts"])))
def test_kat_implicit_casts(case):
    """the restatement takes one type: cast the value set as the reference does (or the input when that fails)"""
    c = KAT["casts"][case]
    vals, vs = pa.array(c["values"], TYPES[c["values_type"]]), pa.array(c["value_set"], TYPES[c["value_set_type"]])
    try:
        vs = vs.cast(vals.type, safe=True)
    except pa.ArrowInvalid:
        vals = vals.cast(vs.type, safe=True)
    want = pa.array(c["expected"], pa.int32() if c["function"] == "index_in" else pa.bool_())
    assert ref.expected(vals, vs, c["behavior"], c["function"]).equals(want)
    assert getattr(pc, c["function"])(pa.array(c["values"], TYPES[c["values_type"]]),
                                      value_set=pa.array(c["value_set"], TYPES[c["value_set_type"]])).equals(want)


@pytest.mark.parametrize("case", range(len(KAT["errors"])))
def test_kat_errors_in_pyarrow(case):
    c = KAT["errors"][case]
    with pytest.raises(pa.ArrowTypeError, match="Array type doesn't match type of values set"):
        pc.is_in(pa.array(c["values"], TYPES[c["values_type"]]), value_set=pa.array(c["value_set"], TYPES[c["value_set_type"]]))


def _f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def _f32(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def random_pair(tname: str, rng, n: int, m: int, null_p=0.1, set_null_p=0.1):
    """values and a value set of one type drawn from a small domain, so matches, misses and duplicates all occur"""
    t = TYPES[tname]
    if tname == "bool":
        dom = [False, True]
    elif tname in STRINGS:
        dom = ["", "a", "ab", "abc", "x" * 40, "x" * 41, "é", "prefix-" * 6 + "1", "prefix-" * 6 + "2"]
    elif tname == "float":
        dom = [0.0, -0.0, 1.5, -2.0, float("inf"), _f32(0x7fc00000), _f32(0x7fc00001), _f32(0xffc00000), 3.0]
    elif tname == "double":
        dom = [0.0, -0.0, 1.5, -2.0, float("-inf"), _f64(0x7ff8000000000000), _f64(0x7ff8000000000001),
               _f64(0xffffffffffffffff), 2.0 ** 60]
    else:
        info = np.iinfo(t.to_pandas_dtype())
        dom = sorted({int(info.min), int(info.max), 0, 1, -1 if info.min < 0 else 2, 7, 100 % (int(info.max) + 1)})
    def draw(k, p):
        out = []
        for _ in range(k):
            v = dom[rng.integers(len(dom))] if rng.random() >= p else None
            out.append(_py(v, t))
        return pa.array(out, t)
    return draw(n, null_p), draw(m, set_null_p)


@pytest.mark.parametrize("tname", list(TYPES))
@pytest.mark.parametrize("behavior", ["match", "skip"])
@pytest.mark.parametrize("function", ["is_in", "index_in"])
def test_against_pyarrow(tname, behavior, function):
    rng = np.random.default_rng(zlib.crc32(f"{tname}/{behavior}/{function}".encode()))
    fn = getattr(pc, function)
    for n, m in [(0, 0), (1, 0), (0, 3), (37, 1), (100, 8), (257, 40), (1000, 300)]:
        vals, vs = random_pair(tname, rng, n, m)
        for v_off, s_off in [(0, 0), (3, 0), (0, 2), (5, 7)]:
            if v_off > n or s_off > m:
                continue
            v, s = vals.slice(v_off), vs.slice(s_off)
            want = fn(v, value_set=s, skip_nulls=behavior == "skip")
            assert ref.expected(v, s, behavior, function).equals(want), (tname, n, m, v_off, s_off)


@pytest.mark.parametrize("tname", ["int64", "double", "string"])
def test_special_sets(tname):
    """an empty set, an all-null set, heavy duplicates, signed zeros and NaN payloads, empty strings"""
    rng = np.random.default_rng(7)
    vals, _ = random_pair(tname, rng, 500, 0)
    t = TYPES[tname]
    dup = pa.concat_arrays([random_pair(tname, rng, 0, 3)[1]] * 200)
    for vs in (pa.array([], t), pa.array([None] * 5, t), dup, dup.slice(17), pa.chunked_array([dup.slice(0, 10), dup.slice(10)])):
        for behavior in ("match", "skip"):
            for function in ("is_in", "index_in"):
                want = getattr(pc, function)(vals, value_set=vs, skip_nulls=behavior == "skip")
                assert ref.expected(vals, vs, behavior, function).equals(want)


def test_float_bit_patterns():
    """-0.0 != +0.0 and a NaN matches only the same payload (UnsignedIntType<8> keys)"""
    vals = pa.array(np.array([0.0, -0.0, np.nan], dtype=np.float64))
    nan2 = np.frombuffer(np.uint64(0x7ff8000000000001).tobytes(), np.float64)[0]
    vs = pa.array(np.array([-0.0, nan2], dtype=np.float64))
    got = ref.expected(vals, vs, "match", "is_in")
    assert got.to_pylist() == [False, True, False]
    assert pc.is_in(vals, value_set=vs).to_pylist() == [False, True, False]


def test_null_slots_are_zero():
    data, valid = ref.set_lookup(pa.array([1, None, 3], pa.int64()), pa.array([3, None], pa.int64()), "emit_null", "index_in")
    assert data.tolist() == [0, 0, 0] and valid.tolist() == [False, False, True]
