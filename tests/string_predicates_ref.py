"""A host restatement, without pyarrow.compute, of the string predicates the device runs (csrc/string_predicates.cu):

  * compare: unsigned bytewise order, a proper prefix first (string_view compare, kernels/scalar_compare.cc:42-72);
  * match_substring / starts_with / ends_with: byte matches (scalar_string_ascii.cc:1221-1307), "" matches everything;
  * match_like: MatchLike::Exec's dispatch (:1533-1588) -- the three classifying regexes, tried in order, then
    MakeLikeRegex (:1456-1497) -- restated with Python `re`, over str for utf8 and over bytes for binary.

Every slot is evaluated, nulls included, over the bytes its offsets span; validity is the AND of the inputs'."""
import re

import numpy as np
import pyarrow as pa

UTF8_TYPES = (pa.string(), pa.large_string())
BINARY_LIKE = (pa.string(), pa.large_string(), pa.binary(), pa.large_binary())

# MatchLikeConstants (scalar_string_ascii.cc:1499-1507)
LIKE_SUBSTRING = r"%+([^%_]*[^\\%_])?%+"
LIKE_STARTS_WITH = r"([^%_]*[^\\%_])?%+"
LIKE_ENDS_WITH = r"%+([^%_]*)"


class InvalidPattern(ValueError):
    """the reference's `Invalid: Invalid regular expression: invalid UTF-8`"""


def slots(arr: pa.Array):
    """the bytes of every slot of a binary-like array, null slots included"""
    wide = arr.type in (pa.large_string(), pa.large_binary())
    bufs = arr.buffers()
    offs = np.frombuffer(bufs[1], np.int64 if wide else np.int32, count=arr.offset + len(arr) + 1)[arr.offset:]
    data = bufs[2].to_pybytes() if bufs[2] is not None else b""
    return [data[int(offs[i]):int(offs[i + 1])] for i in range(len(arr))]


def validity(arr: pa.Array) -> np.ndarray:
    if arr.null_count == 0:
        return np.ones(len(arr), bool)
    return np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), bool)


def order(a: bytes, b: bytes) -> int:
    """-1 / 0 / 1: Python's bytes order is unsigned bytewise, a proper prefix first"""
    return (a > b) - (a < b)


COMPARE = {"equal": lambda c: c == 0, "not_equal": lambda c: c != 0, "greater": lambda c: c > 0,
           "greater_equal": lambda c: c >= 0, "less": lambda c: c < 0, "less_equal": lambda c: c <= 0}


def compare(op: str, left, right):
    """(data, valid) of op(left, right): each side a pa.Array or a scalar given as bytes (None: a null scalar, which
    gives an all-null result whose data bits compare with b"", as UnboxScalar of a null scalar does)"""
    n = len(left) if isinstance(left, pa.Array) else len(right)
    lv = slots(left) if isinstance(left, pa.Array) else [left or b""] * n
    rv = slots(right) if isinstance(right, pa.Array) else [right or b""] * n
    valid = np.ones(n, bool)
    for side in (left, right):
        if isinstance(side, pa.Array):
            valid &= validity(side)
        elif side is None:
            valid[:] = False
    return np.array([COMPARE[op](order(a, b)) for a, b in zip(lv, rv)], bool), valid


def _valid_utf8(b: bytes) -> bool:
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def make_like_regex(pattern):
    """MakeLikeRegex: `%` -> .*, `_` -> ., `\\` escapes the next character (a trailing lone one is dropped), the
    characters .?+*^$\\[{()| escaped.  RE2's `$` is the end of the text; Python's is \\Z.

    RE2 matches in linear time; Python's `re` backtracks, and `.*a.*b.*c` over a long row that fails takes time of the
    row length to the power of the `%` count.  So the same language is written as `^S0(?>.*?S1)...(?>.*?Sk-1).*Sk\\Z`,
    segments Si split at `%`: every middle segment is taken at its leftmost match and never revisited.  That loses no
    match: a segment holds no `%`, so it spans a fixed number of characters, and its leftmost match leaves the most text
    to the segments after it."""
    esc = set(".?+*^$\\[{()|")
    segs, escaped = [[]], False
    for c in pattern:
        if not escaped and c == "%":
            segs.append([])
        elif not escaped and c == "_":
            segs[-1].append(".")
        elif not escaped and c == "\\":
            escaped = True
        else:
            segs[-1].append("\\" + c if c in esc else c)
            escaped = False
    segs = ["".join(s) for s in segs]
    if len(segs) == 1:
        return "(?s:^" + segs[0] + r"\Z)"
    middle = "".join("(?>.*?" + s + ")" for s in segs[1:-1] if s)
    return "(?s:^" + segs[0] + middle + ".*" + segs[-1] + r"\Z)"


def like_plan(pattern: bytes, utf8: bool):
    """(what runs, its pattern): ("match_substring" | "starts_with" | "ends_with", literal bytes) when a classifying
    regex takes the pattern, else ("regex", compiled regex over str (utf8) or bytes (binary)).  Over utf8 a pattern that
    is not valid UTF-8 raises InvalidPattern: the classifying regexes do not match it and the regex does not compile."""
    if utf8:
        if not _valid_utf8(pattern):
            raise InvalidPattern("Invalid regular expression: invalid UTF-8")
        p = pattern.decode("utf-8")
        enc = lambda s: s.encode("utf-8")  # noqa: E731
    else:
        p = pattern.decode("latin-1")  # RE2's Latin-1 mode: one byte, one character
        enc = lambda s: s.encode("latin-1")  # noqa: E731
    for kind, rx in (("match_substring", LIKE_SUBSTRING), ("starts_with", LIKE_STARTS_WITH), ("ends_with", LIKE_ENDS_WITH)):
        m = re.fullmatch(rx, p, re.S)
        if m:
            return kind, enc(m.group(1) or "")
    rx = make_like_regex(p)
    return "regex", re.compile(rx) if utf8 else re.compile(rx.encode("latin-1"))


def match_one(kind: str, s: bytes, pat, utf8: bool) -> bool:
    if kind == "match_substring":
        return pat in s
    if kind == "starts_with":
        return s.startswith(pat)
    if kind == "ends_with":
        return s.endswith(pat)
    return pat.search(s.decode("utf-8") if utf8 else s) is not None


def string_match(function: str, arr: pa.Array, pattern):
    """(data, valid) of function(arr, MatchSubstringOptions(pattern)), ignore_case false"""
    pattern = pattern.encode("utf-8") if isinstance(pattern, str) else bytes(pattern)
    utf8 = arr.type in UTF8_TYPES
    kind, pat = like_plan(pattern, utf8) if function == "match_like" else (function, pattern)
    return np.array([match_one(kind, s, pat, utf8) for s in slots(arr)], bool), validity(arr)


def to_arrow(data: np.ndarray, valid: np.ndarray) -> pa.Array:
    return pa.array(data, pa.bool_(), mask=~valid)


def raw_bits(arr: pa.Array) -> np.ndarray:
    """a boolean result's data bits, slots under nulls included"""
    bits = np.unpackbits(np.frombuffer(arr.buffers()[1], np.uint8), bitorder="little")
    return bits[arr.offset:arr.offset + len(arr)].astype(bool)
