"""The restated sort over utf8 / binary keys (tests/string_sort_oracle.py; ArrayCompareSorter,
kernels/vector_array_sort.cc:144-178) against the reference binary: array_sort_indices on all four base-binary types, both orders and null placements, sliced inputs,
and sort_indices on tables that mix string and numeric keys.  The GPU test of the same inputs checks the device sort
against this restatement."""
import json
import os

import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import string_sort_oracle as sso
from tests.sort_string_cases import (STRING_TYPES, cases, random_bytes, shared_prefix_strings, strings_array,
                                     two_long_identical)
from tests.util import HERE, SEED, random_array

ORDERS = ["ascending", "descending"]
PLACEMENTS = ["at_end", "at_start"]


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
@pytest.mark.parametrize("null_p", [0.0, 0.1, 1.0])
def test_oracle_string_sort_matches_reference(t, null_p):
    for offset in (0, 5):
        arr = strings_array(t, random_bytes(3000, SEED + offset), null_p, SEED + 7, offset=offset)
        for order in ORDERS:
            for placement in PLACEMENTS:
                want = pc.array_sort_indices(arr, order=order, null_placement=placement)
                assert sso.sort_indices(arr, order, placement).equals(want), (t, null_p, offset, order, placement)


@pytest.mark.parametrize("t", [pa.binary(), pa.large_string()], ids=str)
def test_oracle_string_sort_cases(t):
    inputs = [(name, vals, p) for name, vals, p in cases(n_big=(0, 1, 2, 4097))]
    inputs.append(("shared 64 KiB prefix", shared_prefix_strings(SEED), 0.0))
    inputs.append(("two identical 1 MiB strings", two_long_identical(SEED), 0.05))
    for name, vals, null_p in inputs:
        arr = strings_array(t, vals, null_p, SEED, offset=3)
        for order in ORDERS:
            for placement in PLACEMENTS:
                want = pc.array_sort_indices(arr, order=order, null_placement=placement)
                assert sso.sort_indices(arr, order, placement).equals(want), (name, order, placement)


def test_oracle_select_k_and_issue_example():
    a = pa.array([b"\x80", b"a", b"", None, b"a\x00", b"a", b"\xff\x01"])
    assert sso.sort_indices(a).to_pylist() == [2, 1, 5, 4, 0, 6, 3]
    s = pa.array(["b", "a", None, "a"])
    assert sso.select_k_unstable(s, 3, "descending").to_pylist() == [0, 1, 3]


def test_oracle_table_sort_string_and_numeric_keys():
    n = 2000
    cols = {
        "s": strings_array(pa.string(), random_bytes(n, SEED, max_len=3, alphabet=b"xyz"), 0.1, SEED + 1),
        "i": random_array(pa.int64(), n, 0.1, SEED + 2, lo=-3, hi=3),
        "b": strings_array(pa.large_binary(), random_bytes(n, SEED + 3, max_len=2, alphabet=b"\x00\xff"), 0.05, SEED + 4),
    }
    for keys in ([("s", "descending"), ("i", "ascending")], [("i", "descending"), ("b", "ascending"), ("s", "ascending")],
                 [("b", "descending"), ("s", "descending")]):
        for placement in PLACEMENTS:
            want = pc.sort_indices(pa.table(cols), sort_keys=keys, null_placement=placement)
            assert sso.sort_indices_multi(cols, keys, placement).equals(want), (keys, placement)


def test_kat_string_sort():
    with open(os.path.join(HERE, "golden", "kat_sort_strings.json")) as f:
        k = json.load(f)
    for tname in k["types"]:
        for case in k["cases"]:
            arr = pa.array(case["values"], getattr(pa, tname)())
            got = sso.sort_indices(arr, case["order"], case["null_placement"])
            assert got.to_pylist() == case["expected"], (tname, case)
            assert pc.array_sort_indices(arr, order=case["order"], null_placement=case["null_placement"]).to_pylist() == case["expected"]
