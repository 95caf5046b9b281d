"""String predicates (csrc/string_predicates.cu) and string set lookup (csrc/set_lookup.cu) on the device at the byte
lengths where their kernels change path, against the host restatements and pyarrow.compute, data bits under null slots
included, for utf8, large_utf8, binary and large_binary: rows of 0-80 bytes and around 256, 1024, 2048 and 4096 bytes
and 1 MiB; patterns of 1-17 bytes and around 32, 64 and 1024 bytes; occurrences at every start around a lane's search
window; long rows at chosen lanes of a warp, under null slots and in the last partial group; `_` over 1- to 4-byte
code points; character data at every device address mod 8.  The inputs come from string_boundaries."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from tests import set_lookup_ref as sref
from tests import string_boundaries as sb
from tests import string_predicates_ref as ref

pytestmark = pytest.mark.gpu
COMPARES = tuple(ref.COMPARE)
AFFIXES = ("match_substring", "starts_with", "ends_with")
# every offset width on each side, and both mixed pairs
TYPE_PAIRS = [(n, n) for n in sb.TYPES] + [("string", "large_binary"), ("large_string", "binary")]


def check_match(ctx, function, arr: pa.Array, pattern: bytes, align: int = 1):
    got = getattr(bc, function)(sb.upload(ctx, arr, align), pattern).to_arrow()
    data, valid = ref.string_match(function, arr, pattern)
    assert got.equals(ref.to_arrow(data, valid)), (function, arr.type, len(pattern), pattern[:24], align)
    np.testing.assert_array_equal(ref.raw_bits(got), data, err_msg=f"{function} {arr.type} m={len(pattern)}")
    assert got.equals(getattr(pc, function)(arr, pattern))


def check_compare(ctx, op, left, right, align=(1, 1)):
    """each side a pa.Array (uploaded with its character data at 8k + align) or a pa.Scalar"""
    dl = sb.upload(ctx, left, align[0]) if isinstance(left, pa.Array) else left
    dr = sb.upload(ctx, right, align[1]) if isinstance(right, pa.Array) else right
    got = getattr(bc, op)(dl, dr).to_arrow()
    rl = left if isinstance(left, pa.Array) else left.as_buffer().to_pybytes()
    rr = right if isinstance(right, pa.Array) else right.as_buffer().to_pybytes()
    data, valid = ref.compare(op, rl, rr)
    assert got.equals(ref.to_arrow(data, valid)), (op, left.type, right.type, align)
    np.testing.assert_array_equal(ref.raw_bits(got), data, err_msg=f"{op} {left.type} {right.type} {align}")
    assert got.equals(getattr(pc, op)(left, right))


def scalar(row: bytes, t) -> pa.Scalar:
    return pa.scalar(row.decode() if t in ref.UTF8_TYPES else row, t)


def family_arrays(families, t, null_every=0):
    """(bases, variants): every base repeated once per variant, against its variants, all families in one array"""
    bases = [b for b, v in families for _ in v]
    variants = [x for _, v in families for x in v]
    null = None if not null_every else (np.arange(len(variants)) % null_every) == 3
    return sb.array(bases, t), sb.array(variants, t, null)


@pytest.mark.parametrize("lname,rname", TYPE_PAIRS)
def test_compare_families_array_array(ctx, lname, rname):
    """every family of string_boundaries in one array against its bases, both ways round: differences at bytes 0, 7-9,
    255-257, 1023-1025 and the last, proper prefixes, trailing NULs, bytes >= 0x80; equal-length rows of up to 1 MiB are
    the equality rows that take the warp path"""
    lt, rt = sb.TYPES[lname], sb.TYPES[rname]
    utf8 = lt in ref.UTF8_TYPES or rt in ref.UTF8_TYPES
    fams = sb.compare_families(100 + utf8, utf8)
    bl, vr = family_arrays(fams, lt)[0], family_arrays(fams, rt, 11)[1]
    bl_r, vr_l = family_arrays(fams, rt)[0], family_arrays(fams, lt, 11)[1]
    for op in COMPARES:
        check_compare(ctx, op, bl, vr)
        check_compare(ctx, op, vr_l, bl_r)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_compare_families_scalar(ctx, tname):
    """a family's base as the scalar against its variants, on either side: the long side left, right or both"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    lengths = (0, 1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 80) + sb.ROW_LENGTHS[81:] + (sb.MIB,)
    for base, variants in sb.compare_families(200, utf8, lengths):
        arr, s = sb.array(variants, t, (np.arange(len(variants)) % 7) == 5), scalar(base, t)
        for op in COMPARES:
            check_compare(ctx, op, arr, s)
            check_compare(ctx, op, s, arr)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_match_pattern_lengths(ctx, tname):
    """match_substring, starts_with, ends_with and the classified LIKE patterns at every pattern length: occurrences at
    every start around a lane window, at the first and last start and a byte short, the tail changed, m > 1024 and m
    greater than the row"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(300 + len(tname))
    for m in sb.PATTERN_LENGTHS:
        p = sb.pattern(rng, m, utf8)
        rows = sb.substring_texts(rng, p, utf8) + sb.affix_rows(rng, p, utf8)
        arr = sb.array(rows, t, (np.arange(len(rows)) % 13) == 4)
        for f in AFFIXES:
            check_match(ctx, f, arr, p)
        for lp in sb.classified_like(p):
            check_match(ctx, "match_like", arr, lp)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_match_self_overlap_and_head_decoys(ctx, tname):
    t = sb.TYPES[tname]
    for p, rows in sb.self_overlap_cases() + sb.head_decoy_cases():
        arr = sb.array(rows, t)
        for f in AFFIXES:
            check_match(ctx, f, arr, p)
        check_match(ctx, "match_like", arr, b"%" + p + b"%")


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_match_mib_rows(ctx, tname):
    """1 MiB rows: the pattern at the last start, a byte short of it, and at the first start"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(400 + len(tname))
    for m in (1, 8, 9, 64, 65, 1025, 2000):
        p = sb.pattern(rng, m, utf8)
        body = sb.text(rng, sb.MIB - m, utf8)
        last = body + p
        rows = [last, last[:sb.boundary(last, sb.MIB - 1)], p + body, b"x"]
        arr = sb.array(rows, t, [False, False, False, True])
        for f in AFFIXES:
            check_match(ctx, f, arr, p)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_general_like(ctx, tname):
    """patterns no classifying regex takes, over rows on both sides of 1024 bytes in one warp: `_` is one code point of 1
    to 4 bytes over utf8 (also as the last item, after a 3- or 4-byte code point) and one byte over binary"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(500 + len(tname))
    for p in sb.GENERAL_PATTERNS:
        rows = sb.like_rows(rng, p, True) + sb.like_rows(rng, p, utf8)
        assert bc.string_match_plan(p, utf8)[0] == "match_like", p
        check_match(ctx, "match_like", sb.array(rows, t, (np.arange(len(rows)) % 9) == 2), p.encode())


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_warp_layouts(ctx, tname):
    """long rows (taken by the whole warp) mixed with short ones in 32-row groups: 0, 1, 2, 31, 32 per group, at lanes 0
    and 31, under null slots, in the last partial group, and an array whose rows are all long"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(600 + len(tname))
    is_long, null = sb.warp_layout(rng)
    for lng, nul in ((is_long, null), (np.ones(70, bool), (np.arange(70) % 10) == 0)):
        left, right = sb.layout_compare_rows(rng, lng, utf8)
        la, ra = sb.array(left, t, nul), sb.array(right, t)
        for op in COMPARES:
            check_compare(ctx, op, la, ra)
            check_compare(ctx, op, ra, la)
            check_compare(ctx, op, la, scalar(left[int(np.argmax(lng))], t))
        for m in (9, 65, 1100):
            p = sb.pattern(rng, m, utf8)
            arr = sb.array(sb.layout_match_rows(rng, lng, p, utf8), t, nul)
            for f in AFFIXES:
                check_match(ctx, f, arr, p)


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_data_alignment(ctx, tname):
    """character data at every address mod 8, each side of a compare at its own (the multi-difference rows of the
    families included), and under the match functions; and, with the data buffer aligned, slices whose first row
    starts at every byte of a word"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(700 + len(tname))
    lengths = tuple(range(0, 41)) + (255, 256, 257, 1023, 1024, 1025, 1026, 2049)
    fams = sb.compare_families(701, utf8, lengths)
    bases, variants = family_arrays(fams, t, 5)
    pats = [sb.pattern(rng, m, utf8) for m in (1, 7, 8, 9, 17, 65, 1025)]
    texts = sum((sb.substring_texts(rng, p, utf8)[::3] for p in pats), [])
    ones = [b"z"] * 7  # sliced off one at a time, they move the first row's start through a word
    for a in range(8):
        for op in ("equal", "less", "greater_equal"):
            check_compare(ctx, op, bases, variants, (a, (5 * a + 3) % 8))
            check_compare(ctx, op, variants, scalar(fams[-3][0], t), (a, 0))
        whole = sb.array(ones + texts, t)
        for p in pats:
            for f in AFFIXES:
                check_match(ctx, f, whole, p, align=a)
                check_match(ctx, f, whole.slice(a), p, align=0)
        general = sb.array(ones + sb.like_rows(rng, sb.GENERAL_PATTERNS[0], utf8), t).slice(a)
        check_match(ctx, "match_like", general, sb.GENERAL_PATTERNS[0].encode(), align=0)


def set_lookup_data(arr: pa.Array, function: str) -> np.ndarray:
    """the data of an is_in / index_in result, slots under nulls included"""
    if function == "index_in":
        return np.frombuffer(arr.buffers()[1], np.int32, count=arr.offset + len(arr))[arr.offset:]
    return ref.raw_bits(arr)


def check_set_lookup(ctx, values, vs, behavior, function, align):
    got = getattr(bc, function)(sb.upload(ctx, values, align[0]), sb.upload(ctx, vs, align[1]),
                                null_matching_behavior=behavior).to_arrow()
    data, valid = sref.set_lookup(values, vs, behavior, function)
    assert got.equals(sref.to_arrow(data, valid, function)), (function, behavior, values.type, len(vs), align)
    np.testing.assert_array_equal(set_lookup_data(got, function), np.where(valid, data, 0).astype(data.dtype))
    if behavior in ("match", "skip"):
        assert got.equals(getattr(pc, function)(values, value_set=vs, skip_nulls=behavior == "skip"))


@pytest.mark.parametrize("tname", list(sb.TYPES))
def test_set_lookup_alignment(ctx, tname):
    """is_in / index_in over strings of 0-40, 1023-1025 bytes and 1 MiB that differ only at byte 8k - 1, 8k, the last
    byte or in trailing NULs, with the values and the value set at different addresses mod 8, the table in shared memory
    (a few hundred values) and in global memory (over 4096)"""
    t = sb.TYPES[tname]
    utf8 = t in ref.UTF8_TYPES
    rng = np.random.default_rng(800 + len(tname))
    in_set, probes = sb.set_lookup_strings(rng, utf8)
    filler = [b"f%05d" % i for i in range(5000)]
    rows = probes + filler[::7] + [b""]
    values = sb.array(rows, t, (np.arange(len(rows)) % 17) == 6)
    for vs_rows, shared in ((in_set, True), (in_set + filler, False)):
        vs = sb.array(vs_rows, t)
        assert bc.set_lookup_table(sb.upload(ctx, vs))[1] == shared
        for a in range(8):
            align = (a, (3 * a + 5) % 8)
            for function in ("is_in", "index_in"):
                check_set_lookup(ctx, values, vs, "match" if a % 2 else "inconclusive", function, align)
