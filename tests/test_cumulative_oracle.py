"""tests/cumulative_ref.py against the reference's own expected cases (tests/golden/kat_cumulative.json) and against
pyarrow.compute, for every cumulative function over every type, start and null mode; and the CUMULATIVE_OPS table of
the Python binding against the B2CumulativeOp enum of include/arrow_b200.h."""
import json
import os
import shutil
import subprocess
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from arrow_b200 import _cabi as cabi
from tests import cumulative_ref as cr
from tests.test_cabi_enums import ROOT, header_enumerators

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_cumulative.json")
PA_TYPE = {"uint8": pa.uint8(), "int8": pa.int8(), "uint16": pa.uint16(), "int16": pa.int16(), "uint32": pa.uint32(),
           "int32": pa.int32(), "uint64": pa.uint64(), "int64": pa.int64(), "float": pa.float32(), "double": pa.float64()}


def bits_equal(got: pa.Array, want: pa.Array) -> bool:
    """equal types, validity and value bits (so -0.0 differs from 0.0 and NaN equals NaN) at every valid row"""
    if got.type != want.type or len(got) != len(want) or got.null_count != want.null_count:
        return False
    if not np.array_equal(np.asarray(got.is_valid()), np.asarray(want.is_valid())):
        return False
    valid = np.asarray(got.is_valid())
    dt = np.dtype(got.type.to_pandas_dtype())
    g = np.asarray(got.fill_null(0).to_numpy(zero_copy_only=False), dt).view(f"u{dt.itemsize}")
    w = np.asarray(want.fill_null(0).to_numpy(zero_copy_only=False), dt).view(f"u{dt.itemsize}")
    if dt.kind == "f":  # every NaN is the same NaN: payloads are not part of the contract
        gn = np.isnan(np.asarray(got.fill_null(0).to_numpy(zero_copy_only=False), dt))
        wn = np.isnan(np.asarray(want.fill_null(0).to_numpy(zero_copy_only=False), dt))
        return bool(np.array_equal(gn & valid, wn & valid) and np.array_equal(g[valid & ~gn], w[valid & ~wn]))
    return bool(np.array_equal(g[valid], w[valid]))


def _json_values(vals):
    return [float("nan") if v == "NaN" else v for v in vals]


def _kat_cases():
    for c in json.load(open(GOLDEN))["cases"]:
        for t in c["types"]:
            yield pytest.param(c, t, id=f'{c["test"]}-{c["function"]}-{t}')


@pytest.mark.parametrize("case,tname", list(_kat_cases()))
def test_restatement_matches_the_reference_cases(case, tname):
    t = PA_TYPE[tname]
    inputs = [pa.array(_json_values(ch), t) for ch in case["input"]] if case["chunked"] else \
        pa.array(_json_values(case["input"]), t)
    if case["chunked"] and not inputs:
        return
    start = case["start"]
    start = None if start is None else (float(start) if pa.types.is_floating(t) else int(start))
    if case["expected"] == "overflow":
        with pytest.raises(cr.Overflow):
            cr.cumulative(case["function"], inputs, start, case["skip_nulls"])
        return
    out_t = pa.float64() if case["function"] == "cumulative_mean" else t
    want = pa.array(_json_values(case["expected"]), out_t)
    assert bits_equal(cr.cumulative(case["function"], inputs, start, case["skip_nulls"]), want)


def pyarrow_result(name, values, start, skip_nulls):
    """pyarrow.compute over an Array or a ChunkedArray, as one Array; cr.Overflow for its Invalid("overflow")"""
    try:
        out = getattr(pc, name)(values, start=start, skip_nulls=skip_nulls)
    except pa.ArrowInvalid as e:
        assert str(e) == "overflow"
        raise cr.Overflow("overflow")
    return pa.concat_arrays(out.chunks) if isinstance(out, pa.ChunkedArray) else out


def _check(name, chunks, start, skip_nulls):
    try:
        want = pyarrow_result(name, pa.chunked_array(chunks, chunks[0].type), start, skip_nulls)
    except cr.Overflow:
        with pytest.raises(cr.Overflow):
            cr.cumulative(name, chunks, start, skip_nulls)
        return
    got = cr.cumulative(name, chunks, start, skip_nulls)
    assert bits_equal(got, want), (name, chunks, start, skip_nulls, got, want)


def random_column(t: pa.DataType, n: int, rng, null_frac=0.1, small=True):
    dt = np.dtype(t.to_pandas_dtype())
    if dt.kind == "f":
        # dyadic values: every partial sum of a few hundred of them is exact, so the fold order cannot matter
        vals = (rng.integers(-64, 64, n) / 4).astype(dt)
    elif small:
        lo = 0 if dt.kind == "u" else -3
        vals = rng.integers(lo, 4, n).astype(dt)
    else:
        info = np.iinfo(dt)
        vals = rng.integers(int(info.min), int(info.max), n, dtype=dt, endpoint=True)
    return pa.array(vals, t, mask=rng.random(n) < null_frac if null_frac else None)


@pytest.mark.parametrize("t", cr.TYPES, ids=str)
@pytest.mark.parametrize("name", cr.FUNCTIONS)
def test_restatement_matches_pyarrow(name, t):
    rng = np.random.default_rng(zlib.crc32(f"{name}-{t}".encode()))
    for skip_nulls in (False, True):
        for start in (None, 3, 0):
            for null_frac in (0.0, 0.02, 0.3):
                col = random_column(t, 300, rng, null_frac)
                _check(name, [col], start, skip_nulls)
                _check(name, [col.slice(0, 7), col.slice(7, 0), col.slice(7, 100), col.slice(107)], start, skip_nulls)
            # wrap and overflow at full range
            if not pa.types.is_floating(t):
                _check(name, [random_column(t, 50, rng, 0.1, small=False)], start, skip_nulls)


@pytest.mark.parametrize("t", [pa.float32(), pa.float64()], ids=str)
@pytest.mark.parametrize("name", cr.FUNCTIONS)
def test_float_edges_match_pyarrow(name, t):
    edges = [0.0, -0.0, 1.0, -1.0, 2.5, float("inf"), float("-inf"), float("nan"), 1e-30, -1e30]
    rng = np.random.default_rng(7)
    for start in (None, 0.0, -0.0, float("nan"), float("inf"), float("-inf")):
        for skip_nulls in (False, True):
            for _ in range(20):
                vals = rng.choice(edges, 12)
                col = pa.array(vals, t, mask=rng.random(12) < 0.15)
                _check(name, [col], start, skip_nulls)
    # the defaults: max starts at the smallest positive normal, min at the largest finite value
    _check("cumulative_max", [pa.array([-5.0], t)], None, False)
    _check("cumulative_min", [pa.array([float("inf")], t)], None, False)
    _check("cumulative_min", [pa.array([0.0, -0.0, 0.0], t)], None, False)
    _check("cumulative_max", [pa.array([-0.0, 0.0, -0.0], t)], 0.0, False)


@pytest.mark.parametrize("name", ["cumulative_sum_checked", "cumulative_prod_checked"])
def test_checked_overflow_positions_match_pyarrow(name):
    big = 2 ** 62
    cases = [
        [1, None, big, big],          # after the first null, nothing is combined: no error
        [big, big, None],             # before it: the error
        [big, 4, 0],                  # prod: the final product is 0 but a prefix overflowed
        [-big, -big, -1],
        [2 ** 63 - 1],
    ]
    for vals in cases:
        for skip_nulls in (False, True):
            _check(name, [pa.array(vals, pa.int64())], None, skip_nulls)
            _check(name, [pa.array(vals, pa.int64())], 2, skip_nulls)
    # a start that overflows on the first row
    _check(name, [pa.array([127], pa.int8())], 1 if "sum" in name else 2, False)
    _check(name, [pa.array([1, 1], pa.uint8())], 255, False)


def test_starts_that_fail_to_cast_raise_the_reference_texts():
    # the binding casts `start` on the host with pyarrow's safe cast; these are the texts the reference raises
    for name in ("cumulative_sum", "cumulative_prod", "cumulative_min", "cumulative_max"):
        for value, t, text in ((1.5, pa.int64(), "Float value 1.500000 was truncated converting to int64"),
                               (1000, pa.int8(), "Integer value 1000 not in range: -128 to 127"),
                               (-1, pa.uint32(), "Integer value -1 not in range: 0 to 4294967295")):
            with pytest.raises(pa.ArrowInvalid, match=text):
                getattr(pc, name)(pa.array([1], t), start=value)
            with pytest.raises(pa.ArrowInvalid, match=text):
                pa.scalar(value).cast(t, safe=True)
    # a null start contributes the bits it carries
    _check("cumulative_sum", [pa.array([1, 2], pa.int64())], pa.scalar(None, pa.int64()), False)
    # cumulative_mean ignores start
    _check("cumulative_mean", [pa.array([1, 2], pa.int64())], 100, False)


@pytest.mark.parametrize("t", [pa.float16(), pa.bool_(), pa.decimal128(5, 2), pa.duration("s")], ids=str)
def test_types_without_a_kernel(t):
    vals = pa.array([np.float16(1)], t) if t == pa.float16() else pa.array([True] if t == pa.bool_() else [1], t)
    for name in cr.FUNCTIONS:
        with pytest.raises(pa.ArrowNotImplementedError, match=f"Function '{name}' has no kernel matching input types"):
            getattr(pc, name)(vals)


def test_cumulative_ops_match_the_header_enum(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    members = header_enumerators()["B2CumulativeOp"]
    src = tmp_path / "enums.c"
    src.write_text('#include <stdio.h>\n#include "arrow_b200.h"\nint main(void) {\n'
                   + "\n".join(f'printf("{e} %lld\\n", (long long){e});' for e in members) + "\nreturn 0; }\n")
    exe = tmp_path / "enums"
    subprocess.check_call(["gcc", "-std=c11", "-I", f"{ROOT}/include", str(src), "-o", str(exe)])
    got = {k: int(v) for k, v in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                       check=True).stdout.splitlines())}
    assert {"B2_" + k.upper(): v for k, v in cabi.CUMULATIVE_OPS.items()} == got
    assert set(cabi.CUMULATIVE_OPS) == set(cr.FUNCTIONS)
