"""The host restatements of the string predicates (string_predicates_ref) and of set lookup (set_lookup_ref) against
pyarrow.compute on every input of string_boundaries -- rows and patterns at the lengths where the device kernels change
path, code points of 1 to 4 bytes, NULs and bytes >= 0x80 -- for all four binary-like types, so the device tests
compare against a reference pinned on exactly these inputs.  CPU only."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import set_lookup_ref as sref
from tests import string_boundaries as sb
from tests import string_predicates_ref as ref

COMPARES = tuple(ref.COMPARE)


def check_match(function, arr: pa.Array, pattern):
    want = getattr(pc, function)(arr, pattern)
    data, valid = ref.string_match(function, arr, pattern)
    assert ref.to_arrow(data, valid).equals(want), (function, arr.type, pattern[:40], len(pattern))
    np.testing.assert_array_equal(ref.raw_bits(want), data, err_msg=f"{function} {arr.type} {len(pattern)}")


def check_compare(op, left, right, rl, rr):
    """left / right as given to pyarrow; rl / rr as given to the restatement"""
    want = getattr(pc, op)(left, right)
    data, valid = ref.compare(op, rl, rr)
    assert ref.to_arrow(data, valid).equals(want), (op, left.type, right.type)
    np.testing.assert_array_equal(ref.raw_bits(want), data, err_msg=op)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_compare_families(tname):
    """every family of string_boundaries: the base against its variants, both ways round, as arrays and as scalars"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    for base, variants in sb.compare_families(10, utf8):
        arr = sb.array(variants, t, [False] * (len(variants) - 1) + [True])
        bases = sb.array([base] * len(variants), t)
        s = pa.scalar(base.decode() if utf8 else base, t)
        for op in COMPARES:
            check_compare(op, bases, arr, bases, arr)
            check_compare(op, arr, bases, arr, bases)
            check_compare(op, arr, s, arr, base)
            check_compare(op, s, arr, base, arr)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_substring_prefix_suffix(tname):
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(20 + len(tname))
    for m in sb.PATTERN_LENGTHS:
        p = sb.pattern(rng, m, utf8)
        arr = sb.array(sb.substring_texts(rng, p, utf8) + sb.affix_rows(rng, p, utf8), t)
        for f in ("match_substring", "starts_with", "ends_with"):
            check_match(f, arr, p)
        for lp in sb.classified_like(p):
            check_match("match_like", arr, lp)
    for p, rows in sb.self_overlap_cases() + sb.head_decoy_cases():
        arr = sb.array(rows, t)
        for f in ("match_substring", "starts_with", "ends_with"):
            check_match(f, arr, p)
        check_match("match_like", arr, b"%" + p + b"%")


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_general_like(tname):
    """the patterns no classifying regex takes, over rows on both sides of 1024 bytes; `_` is one code point over utf8
    (1 to 4 bytes) and one byte over binary"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(30 + len(tname))
    for p in sb.GENERAL_PATTERNS:
        assert ref.like_plan(p.encode(), utf8)[0] == "regex", p
        rows = sb.like_rows(rng, p, True) + sb.like_rows(rng, p, utf8)  # the utf8 instances too, over binary
        check_match("match_like", sb.array(rows, t), p.encode())


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_warp_layouts(tname):
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(40 + len(tname))
    is_long, null = sb.warp_layout(rng)
    left, right = sb.layout_compare_rows(rng, is_long, utf8)
    la, ra = sb.array(left, t, null), sb.array(right, t)
    for op in COMPARES:
        check_compare(op, la, ra, la, ra)
    for m in (9, 65, 1100):
        p = sb.pattern(rng, m, utf8)
        arr = sb.array(sb.layout_match_rows(rng, is_long, p, utf8), t, null)
        for f in ("match_substring", "starts_with", "ends_with"):
            check_match(f, arr, p)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_set_lookup_strings(tname):
    """is_in / index_in over strings differing only at byte 8k - 1, 8k, the last byte or in trailing NULs, with value
    sets on both sides of the 4096 distinct values the device stages in shared memory"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(50 + len(tname))
    in_set, probes = sb.set_lookup_strings(rng, utf8)
    filler = [b"f%05d" % i for i in range(5000)]
    values = sb.array(probes + filler[::7] + [b""], t, [False] * (len(probes) + len(filler[::7])) + [True])
    for vs_rows in (in_set, in_set + filler):
        vs = sb.array(vs_rows, t)
        for function in ("is_in", "index_in"):
            for behavior in ("match", "skip"):
                data, valid = sref.set_lookup(values, vs, behavior, function)
                want = getattr(pc, function)(values, value_set=vs, skip_nulls=behavior == "skip")
                assert sref.to_arrow(data, valid, function).equals(want), (function, behavior, len(vs_rows))
