"""The op-code and kind tables of the Python binding against the enums of include/arrow_b200.h, as the C compiler sees
them, and the options that call_function accepts against the direct call."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from arrow_b200 import _cabi as cabi
from arrow_b200 import compute as bc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# table name: (the table, the C enum it mirrors, the enumerator of each key)
TABLES = {
    "ARITH_OPS": (cabi.ARITH_OPS, "B2ArithOp", lambda k: "B2_" + k.upper()),
    "COMPARE_OPS": (cabi.COMPARE_OPS, "B2CompareOp", lambda k: "B2_" + k.upper()),
    "STRING_MATCH": (cabi.STRING_MATCH, "B2StringMatchKind", lambda k: "B2_MATCH_" + k.removeprefix("match_").upper()),
    "BOOLEAN_OPS": (cabi.BOOLEAN_OPS, "B2BooleanOp", lambda k: "B2_BOOL_" + k.upper()),
    "VALIDITY_OPS": (cabi.VALIDITY_OPS, "B2ValidityOp", lambda k: "B2_" + k.upper()),
    "TEMPORAL_KINDS": (cabi.TEMPORAL_KINDS, "B2TemporalKind", lambda k: "B2_TEMPORAL_" + k.upper()),
    "TIME_UNITS": (cabi.TIME_UNITS, "B2TimeUnit", {"s": "B2_SECOND", "ms": "B2_MILLI", "us": "B2_MICRO", "ns": "B2_NANO"}.get),
    "TEMPORAL_FIELDS": (cabi.TEMPORAL_FIELDS, "B2TemporalField", lambda k: "B2_FIELD_" + k.upper()),
    "HASH_AGG_KINDS": (cabi.HASH_AGG_KINDS, "B2HashAggKind", lambda k: "B2_" + k.upper()),
    "JOIN_TYPES": (bc.JOIN_TYPES, "B2JoinType", lambda k: "B2_JOIN_" + k.upper().replace(" ", "_")),
}


def header_enumerators():
    """{enum name: [enumerator, ...]} of every typedef'd enum in the header"""
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "arrow_b200.h")).read(), flags=re.S)
    return {name: re.findall(r"\b(B2_\w+)\s*=", body) for name, body in re.findall(r"typedef enum (\w+)\s*\{(.*?)\}", text, re.S)}


def test_tables_match_the_header_enums(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    enums = header_enumerators()
    lines = [f'printf("{e} %lld\\n", (long long){e});' for members in enums.values() for e in members]
    lines.append('printf("B2TemporalType %zu\\n", sizeof(B2TemporalType));')
    lines += [f'printf("B2TemporalType.{f} %zu\\n", offsetof(B2TemporalType, {f}));' for f, _ in cabi.B2TemporalType._fields_]
    src = tmp_path / "enums.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "arrow_b200.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0; }\n")
    exe = tmp_path / "enums"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = {k: int(v) for k, v in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())}
    for table_name, (table, enum, enumerator) in TABLES.items():
        want = {e: got[e] for e in enums[enum]}
        mirrored = {enumerator(k): v for k, v in table.items()}
        assert mirrored == want, f"{table_name} differs from {enum}: {mirrored} vs {want}"
    assert got["B2TemporalType"] == C.sizeof(cabi.B2TemporalType)
    for f, _ in cabi.B2TemporalType._fields_:
        assert got[f"B2TemporalType.{f}"] == getattr(cabi.B2TemporalType, f).offset, f"B2TemporalType.{f}"


def _same(got, want):
    if isinstance(want, tuple):
        assert len(got) == len(want)
        for g, w in zip(got, want):
            _same(g, w)
    elif isinstance(want, pa.Scalar):
        assert got.equals(want), (got, want)
    else:
        assert got.to_arrow().equals(want.to_arrow()), (got.to_arrow(), want.to_arrow())


@pytest.mark.gpu
def test_call_function_options_match_the_direct_call(ctx):
    """every registry function that takes options, given them as a pyarrow Options object and as a dict"""
    from arrow_b200 import DeviceArray
    rng = np.random.default_rng(7)
    n = 1000
    ints = DeviceArray.from_arrow(pa.array(rng.integers(-50, 50, n), pa.int64(), mask=rng.random(n) < 0.1), ctx)
    floats = DeviceArray.from_arrow(pa.array(np.where(rng.random(n) < 0.05, np.nan, rng.normal(size=n)), mask=rng.random(n) < 0.1), ctx)
    mask = DeviceArray.from_arrow(pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1), ctx)
    idx = DeviceArray.from_arrow(pa.array(rng.integers(0, n, 200), pa.int32()), ctx)
    words = DeviceArray.from_arrow(pa.array([None if i % 13 == 0 else f"w{i % 37}ab" for i in range(n)]), ctx)
    stamps = DeviceArray.from_arrow(pa.array(rng.integers(0, 2 ** 40, n) * 1000, pa.timestamp("ms")), ctx)
    value_set = pa.array([1, 2, None, 40], pa.int64())
    cases = {  # name: ([args], Options, dict, direct call)
        "cast": ([ints], pc.CastOptions.unsafe(pa.int8()), {"target_type": pa.int8(), "safe": False},
                 lambda: bc.cast(ints, pa.int8(), safe=False)),
        "filter": ([ints, mask], pc.FilterOptions("emit_null"), {"null_selection_behavior": "emit_null"},
                   lambda: bc.filter(ints, mask, "emit_null")),
        "take": ([ints, idx], pc.TakeOptions(boundscheck=False), {"boundscheck": False}, lambda: bc.take(ints, idx, False)),
        "array_sort_indices": ([floats], pc.ArraySortOptions("descending", null_placement="at_start"),
                               {"order": "descending", "null_placement": "at_start"},
                               lambda: bc.array_sort_indices(floats, "descending", "at_start")),
        "sort_indices": ([floats], pc.SortOptions([("x", "descending")], null_placement="at_start"),
                         {"sort_keys": [("x", "descending")], "null_placement": "at_start"},
                         lambda: bc.array_sort_indices(floats, "descending", "at_start")),
        "select_k_unstable": ([ints], pc.SelectKOptions(7, [("x", "descending")]), {"k": 7, "sort_keys": [("x", "descending")]},
                              lambda: bc.select_k_unstable(ints, 7, [("x", "descending")])),
        "dictionary_encode": ([ints], pc.DictionaryEncodeOptions("encode"), {"null_encoding": "encode"},
                              lambda: bc.dictionary_encode(ints, "encode")),
        "count_distinct": ([ints], pc.CountOptions("all"), {"mode": "all"}, lambda: bc.count_distinct(ints, "all")),
        "count": ([ints], pc.CountOptions("only_null"), {"mode": "only_null"}, lambda: bc.count(ints, "only_null")),
        "is_null": ([floats], pc.NullOptions(nan_is_null=True), {"nan_is_null": True}, lambda: bc.is_null(floats, True)),
        "is_in": ([ints], None, {"value_set": value_set, "skip_nulls": True}, lambda: bc.is_in(ints, value_set, True)),
        "index_in": ([ints], None, {"value_set": value_set, "null_matching_behavior": "emit_null"},
                     lambda: bc.index_in(ints, value_set, null_matching_behavior="emit_null")),
        "day_of_week": ([stamps], pc.DayOfWeekOptions(count_from_zero=False, week_start=3),
                        {"count_from_zero": False, "week_start": 3}, lambda: bc.day_of_week(stamps, False, 3)),
        "variance": ([ints], pc.VarianceOptions(ddof=1, min_count=3), {"ddof": 1, "min_count": 3},
                     lambda: bc.variance(ints, ddof=1, min_count=3)),
        "stddev": ([ints], pc.VarianceOptions(ddof=1, skip_nulls=False), {"ddof": 1, "skip_nulls": False},
                   lambda: bc.stddev(ints, ddof=1, skip_nulls=False)),
        "skew": ([ints], pc.SkewOptions(biased=False), {"biased": False}, lambda: bc.skew(ints, biased=False)),
        "kurtosis": ([ints], pc.SkewOptions(biased=False, min_count=5), {"biased": False, "min_count": 5},
                     lambda: bc.kurtosis(ints, biased=False, min_count=5)),
    }
    cases["array_filter"] = cases["filter"]
    cases["array_take"] = cases["take"]
    for name in ("match_substring", "starts_with", "ends_with", "match_like"):
        cases[name] = ([words], pc.MatchSubstringOptions("%ab"), {"pattern": "%ab", "ignore_case": False},
                       (lambda f: lambda: f(words, "%ab"))(getattr(bc, name)))
    for name in ("sum", "mean", "min_max", "min", "max"):
        cases[name] = ([ints], pc.ScalarAggregateOptions(skip_nulls=False, min_count=2), {"skip_nulls": False, "min_count": 2},
                       (lambda f: lambda: f(ints, skip_nulls=False, min_count=2))(getattr(bc, name)))
    taking_options = {name for name, (_, adapt) in bc._REGISTRY.items() if adapt is not None}
    assert set(cases) == taking_options
    for name, (args, options, keywords, direct) in cases.items():
        want = direct()
        if options is not None:  # pyarrow's SetLookupOptions cannot carry the value set through its repr
            _same(bc.call_function(name, args, options), want)
        _same(bc.call_function(name, args, keywords), want)
