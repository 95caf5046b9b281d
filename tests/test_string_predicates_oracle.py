"""The host restatement of the string predicates (string_predicates_ref) against the reference's own expected outputs
(tests/golden/kat_string_predicates.json) and against pyarrow.compute on seeded random strings and random LIKE patterns,
for all four binary-like types.  This pins MatchLike's dispatch quirks: backslashes on the fast paths, `_` over utf8
versus binary, `%` across newlines and the invalid-UTF-8 error.  CPU only."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import string_predicates_ref as ref

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_string_predicates.json")))
TYPES = {"string": pa.string(), "large_string": pa.large_string(), "binary": pa.binary(), "large_binary": pa.large_binary()}
COMPARES = tuple(ref.COMPARE)
MATCHES = ("match_substring", "starts_with", "ends_with", "match_like")
# the pattern alphabet: wildcards, escapes, a newline, a two-byte code point and regex metacharacters; for binary also
# a NUL and a byte that is not UTF-8
PIECES = ["a", "b", "ab", "%", "_", "\\", "\n", "é", ".", "*", "(", "[", "$", "^", "|", "+", "?", "{"]
BINARY_PIECES = [b"\x00", b"\xfc"]


def kat_value(v, t):
    """KAT strings are JSON text; binary values may carry bytes as {"hex": "..."}"""
    if isinstance(v, dict):
        return bytes.fromhex(v["hex"])
    if v is not None and t in (pa.binary(), pa.large_binary()):
        return v.encode("utf-8")
    return v


def kat_pattern(p):
    return bytes.fromhex(p["hex"]) if isinstance(p, dict) else p


def random_strings(rng, n, t, maxlen=8, null_p=0.1):
    pieces = [p.encode() for p in PIECES] + (BINARY_PIECES if t not in ref.UTF8_TYPES else [])
    vals = [b"".join(pieces[k] for k in rng.integers(0, len(pieces), rng.integers(0, maxlen + 1))) for _ in range(n)]
    if t in ref.UTF8_TYPES:
        vals = [v.decode("utf-8") for v in vals]
    return pa.array(vals, t, mask=rng.random(n) < null_p)


def random_pattern(rng, t, maxlen=5):
    pieces = [p.encode() for p in PIECES] + (BINARY_PIECES if t not in ref.UTF8_TYPES else [])
    return b"".join(pieces[k] for k in rng.integers(0, len(pieces), rng.integers(0, maxlen + 1)))


@pytest.mark.parametrize("case", range(len(KAT["match"])))
def test_kat_match(case):
    c = KAT["match"][case]
    for tname in c["types"]:
        t = TYPES[tname]
        arr = pa.array([kat_value(v, t) for v in c["input"]], t)
        pattern = kat_pattern(c["pattern"])
        if c.get("ignore_case"):
            # not on the device: the host result still follows the reference
            want = pa.array(c["expected"], pa.bool_())
            assert getattr(pc, c["function"])(arr, pattern, ignore_case=True).equals(want), (c, tname)
            continue
        if "error" in c:
            with pytest.raises(ref.InvalidPattern, match=c["error"]):
                ref.string_match(c["function"], arr, pattern)
            continue
        got = ref.to_arrow(*ref.string_match(c["function"], arr, pattern))
        assert got.equals(pa.array(c["expected"], pa.bool_())), (c, tname, got)


@pytest.mark.parametrize("case", range(len(KAT["compare"])))
def test_kat_compare(case):
    c = KAT["compare"][case]
    for tname in c["types"]:
        t = TYPES[tname]
        arr = pa.array([kat_value(v, t) for v in c["input"]], t)
        scalar = kat_value(c["scalar"], pa.binary())
        got = ref.to_arrow(*ref.compare(c["function"], arr, scalar))
        assert got.equals(pa.array(c["expected"], pa.bool_())), (c, tname, got)


@pytest.mark.parametrize("tname", list(TYPES))
def test_random_like_against_pyarrow(tname):
    """random strings and random LIKE patterns over the pattern alphabet: the restatement's data and validity match
    pyarrow's, and so does its refusal of an invalid UTF-8 pattern over utf8"""
    t = TYPES[tname]
    rng = np.random.default_rng(1000 + len(tname))
    arr = random_strings(rng, 300, t)
    for _ in range(400):
        p = random_pattern(rng, t)
        try:
            want = pc.match_like(arr, p)
        except pa.ArrowInvalid as e:
            assert "invalid UTF-8" in str(e)
            with pytest.raises(ref.InvalidPattern):
                ref.string_match("match_like", arr, p)
            continue
        data, valid = ref.string_match("match_like", arr, p)
        assert ref.to_arrow(data, valid).equals(want), (tname, p)
        np.testing.assert_array_equal(ref.raw_bits(want), data, err_msg=repr(p))


@pytest.mark.parametrize("tname", list(TYPES))
@pytest.mark.parametrize("function", MATCHES[:3])
def test_random_byte_matches_against_pyarrow(tname, function):
    t = TYPES[tname]
    rng = np.random.default_rng(2000 + len(tname) + MATCHES.index(function))
    arr = random_strings(rng, 300, t)
    for _ in range(100):
        p = random_pattern(rng, t, 3)
        want = getattr(pc, function)(arr, p)
        data, valid = ref.string_match(function, arr, p)
        assert ref.to_arrow(data, valid).equals(want), (tname, function, p)
        np.testing.assert_array_equal(ref.raw_bits(want), data)


@pytest.mark.parametrize("lname", list(TYPES))
@pytest.mark.parametrize("rname", list(TYPES))
def test_random_compares_against_pyarrow(lname, rname):
    """mixed types compare their bytes (the reference casts both to CommonBinary first); data bits under nulls too"""
    rng = np.random.default_rng(3000 + 7 * len(lname) + len(rname))
    left, right = random_strings(rng, 300, TYPES[lname], 4), random_strings(rng, 300, TYPES[rname], 4)
    scalar = ref.slots(right)[0]
    for op in COMPARES:
        want = getattr(pc, op)(left, right)
        data, valid = ref.compare(op, left, right)
        assert ref.to_arrow(data, valid).equals(want)
        np.testing.assert_array_equal(ref.raw_bits(want), data)
        s = pa.scalar(scalar.decode("utf-8") if TYPES[rname] in ref.UTF8_TYPES else scalar, TYPES[rname])
        for args, refargs in (((left, s), (left, scalar)), ((s, left), (scalar, left))):
            want = getattr(pc, op)(*args)
            data, valid = ref.compare(op, *refargs)
            assert ref.to_arrow(data, valid).equals(want)
            np.testing.assert_array_equal(ref.raw_bits(want), data)
        want = getattr(pc, op)(left, pa.scalar(None, TYPES[rname]))
        data, valid = ref.compare(op, left, None)
        assert ref.to_arrow(data, valid).equals(want)
        np.testing.assert_array_equal(ref.raw_bits(want), data)


def test_like_dispatch_examples():
    """the consequences of MatchLike's dispatch, each checked against pyarrow"""
    cases = [
        (pa.string(), ["a\\b", "ab"], "%a\\b%", [True, False], "match_substring"),
        (pa.string(), ["abc\\", "abc"], "%abc\\", [True, False], "ends_with"),
        (pa.string(), ["abc\\\\", "abc\\"], "%abc\\\\", [True, False], "ends_with"),
        (pa.string(), ["é", "e"], "_", [True, True], "regex"),
        (pa.binary(), [b"\xc3\xa9", b"e"], "_", [False, True], "regex"),
        (pa.string(), ["x\ny", "xy"], "%\n%", [True, False], "match_substring"),
        (pa.string(), ["a\nb", "ab"], "a_b", [True, False], "regex"),
        (pa.binary(), [b"\xc3\xa9b", b"b"], b"%\xa9b", [True, False], "ends_with"),
    ]
    for t, vals, p, want, kind in cases:
        arr = pa.array(vals, t)
        assert pc.match_like(arr, p).to_pylist() == want, (t, p)
        assert ref.string_match("match_like", arr, p)[0].tolist() == want, (t, p)
        pb = p.encode() if isinstance(p, str) else p
        assert ref.like_plan(pb, t in ref.UTF8_TYPES)[0] == kind, (t, p)
    with pytest.raises(pa.ArrowInvalid, match="invalid UTF-8"):
        pc.match_like(pa.array(["a"]), b"%\xa9b%")
    with pytest.raises(ref.InvalidPattern):
        ref.like_plan(b"%\xa9b%", True)
