"""The temporal restatement (temporal_ref) against pyarrow.compute: every field x type x unit x zone form and every cast
pair x safety flag, on seeded full-range values plus the edge list (±0 / ±1 around midnight and 1970, leap days in
1900, 2000 and 2100, INT32 / INT64 min and max, exact multiples of a day far below 1970)."""
import json
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import temporal_ref as ref

TYPES = ref.type_variants()
CAST_TYPES = TYPES + [pa.int32(), pa.int64()]


def inputs(t, n=2000, seed=11):
    return np.concatenate([ref.edge_values(t), ref.random_values(t, n, seed)])


@pytest.mark.parametrize("t", TYPES, ids=str)
@pytest.mark.parametrize("field", ref.FIELDS)
def test_fields_match_pyarrow(field, t):
    v = inputs(t)
    arr = ref.to_arrow(v, None, t)
    if not ref.accepts(field, t):
        with pytest.raises(pa.ArrowNotImplementedError):
            pc.call_function(field, [arr])
        return
    want = pc.call_function(field, [arr]).to_numpy(zero_copy_only=False)
    got = np.asarray(ref.field(field, v, t), want.dtype)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("t", [pa.date32(), pa.date64(), pa.timestamp("s", "+05:30"), pa.timestamp("ns")], ids=str)
@pytest.mark.parametrize("week_start", range(1, 8))
@pytest.mark.parametrize("count_from_zero", [True, False])
def test_day_of_week_options(t, week_start, count_from_zero):
    v = inputs(t, 500)
    want = pc.day_of_week(ref.to_arrow(v, None, t), count_from_zero=count_from_zero, week_start=week_start)
    np.testing.assert_array_equal(ref.field("day_of_week", v, t, week_start, count_from_zero), want.to_numpy())


def test_documented_wraps():
    """the reference's answers far from 1970, which only the 32-bit day count and 16-bit year explain"""
    s = pa.timestamp("s")
    for value, ymd in ((2 ** 62, (26826, 1, 29)), (10 ** 12, (-31878, 9, 27)), (-(2 ** 40) * 86400, (1969, 12, 31))):
        got = tuple(int(ref.field(f, [value], s)[0]) for f in ("year", "month", "day"))
        assert got == ymd
    d = pa.date32()
    assert [int(ref.field(f, [2 ** 31 - 1], d)[0]) for f in ("year", "month", "day")] == [20599, 6, 22]
    assert [int(ref.field(f, [-2 ** 31], d)[0]) for f in ("year", "month", "day")] == [20599, 6, 23]


@pytest.mark.parametrize("src", CAST_TYPES, ids=str)
def test_casts_match_pyarrow(src):
    v = inputs(src, 300, 9)
    valid = np.random.default_rng(9).random(len(v)) < 0.9
    arr = ref.to_arrow(v, valid, src)
    for dst in CAST_TYPES:
        if src == dst or (src in (pa.int32(), pa.int64()) and dst in (pa.int32(), pa.int64())):
            continue
        for truncate, overflow in ((False, False), (True, False), (False, True), (True, True)):
            opts = pc.CastOptions(dst, allow_time_truncate=truncate, allow_time_overflow=overflow)
            try:
                want, want_err = pc.cast(arr, options=opts), None
            except (pa.ArrowInvalid, pa.ArrowNotImplementedError) as e:
                want, want_err = None, (type(e), str(e))
            try:
                got, got_err = ref.cast(v, valid, src, dst, truncate, overflow), None
            except ref.CastError as e:
                got, got_err = None, (pa.ArrowInvalid, str(e))
            except NotImplementedError as e:
                got, got_err = None, (pa.ArrowNotImplementedError, str(e))
            assert got_err == want_err, (src, dst, truncate, overflow)
            if want is not None:
                w = np.asarray(want.view(pa.int32() if dst.bit_width == 32 else pa.int64()).fill_null(0))
                np.testing.assert_array_equal(got[valid], w[valid], err_msg=f"{src} -> {dst}")


def test_unsafe_division_truncates_toward_zero():
    got = ref.cast([-1500, 1500], [True, True], pa.timestamp("ms"), pa.timestamp("s"), allow_time_truncate=True)
    assert got.tolist() == [-1, 1]
    assert pc.cast(pa.array([-1500, 1500], pa.timestamp("ms")), pa.timestamp("s"), safe=False).cast(pa.int64()).to_pylist() == [-1, 1]


def test_timestamp_to_date_and_time_floor():
    ms = pa.timestamp("ms")
    assert ref.cast([-1], [True], ms, pa.date32()).tolist() == [-1]
    assert ref.cast([-1], [True], ms, pa.time32("s"), allow_time_truncate=True).tolist() == [86399]


def _parse_type(s: str) -> pa.DataType:
    m = re.fullmatch(r"timestamp\[(\w+)(?:, tz=(.+))?\]", s)
    return pa.timestamp(m.group(1), m.group(2))


def test_reference_expected_outputs():
    """the restatement reproduces the expected outputs of the reference's own tests (tests/golden/kat_temporal.json)"""
    kat = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_temporal.json")))
    f = kat["fields"]
    times = [None if s is None else int(np.datetime64(s.replace(" ", "T"), "ns").astype(np.int64)) for s in f["times"]]
    valid = np.array([x is not None for x in times])
    v = np.array([0 if x is None else x for x in times], np.int64)
    t = pa.timestamp("ns")
    for name, want in f["expected"].items():
        got = ref.field(name, v, t)
        assert [x for x, ok in zip(got.tolist(), valid) if ok] == [w for w in want if w is not None], name
    for case in kat["casts"]:
        src, dst = _parse_type(case["from"]), _parse_type(case["to"])
        cvalid = np.array([x is not None for x in case["values"]])
        cv = np.array([0 if x is None else x for x in case["values"]], np.int64)
        if "error" in case:
            with pytest.raises(ref.CastError, match=case["error"]):
                ref.cast(cv, cvalid, src, dst, case.get("allow_time_truncate", False))
            continue
        got = ref.cast(cv, cvalid, src, dst, case.get("allow_time_truncate", False))
        assert [x for x, ok in zip(got.tolist(), cvalid) if ok] == [w for w in case["expected"] if w is not None], case
