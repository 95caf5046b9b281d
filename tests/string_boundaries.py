"""Seeded inputs for the string predicates and the string set lookup at the byte lengths where their kernels change path
(csrc/string_predicates.cu, csrc/set_lookup.cu, the byte helpers of csrc/common.cuh), shared by the CPU check of the host
restatement (test_string_boundaries_oracle.py) and the device tests (test_gpu_string_boundaries.py).

  * 8-byte loads: first_diff, find_in, hash_bytes and bytes_equal read a row 8 bytes at a time, masking the tail and
    reading a second word when an unaligned load crosses one -- lengths 0-80, differences at bytes 7 / 8 / 9.
  * kLongRow = 1024: a row with more bytes of work leaves its lane and the warp takes it (warp_first_diff 256 bytes per
    step; warp_find_in with lane windows of kWindow = 64 starts, 32 * 64 = 2048 starts per step) -- lengths 1023-1026,
    2047-2049, 4095-4097, occurrences at every start around a lane window, long rows at chosen lanes of a 32-row group.
  * find_in matches a pattern of <= 8 bytes on its 64-bit head alone and verifies a longer one past byte 8.
  * match_segment: over utf8 `_` takes 1, 2, 3 or 4 bytes by the lead byte.

Everything is bytes; a generator for utf8 input makes valid UTF-8 (utf8=True), one for binary may use any byte."""
import numpy as np
import pyarrow as pa

MIB = 1 << 20
ROW_LENGTHS = tuple(range(81)) + (255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 1026, 2047, 2048, 2049,
                                  4095, 4096, 4097)  # 64 * 32 * k +- 1 for k = 1, 2 included
PATTERN_LENGTHS = tuple(range(1, 18)) + (31, 32, 33, 63, 64, 65, 66, 100, 1023, 1024, 1025, 1026, 2000)
DIFF_AT = (0, 7, 8, 9, 255, 256, 257, 1023, 1024, 1025)  # and len - 1
WINDOW = 64      # kWindow

# code points at the encoding boundaries: 1, 2, 2, 3, 3, 4, 4 bytes
BOUNDARY_CPS = ("\u007f", "\u0080", "\u07ff", "\u0800", "\uffff", "\U00010000", "\U0010ffff")
CP_BYTES = tuple(c.encode() for c in BOUNDARY_CPS)
# filler alphabet of the rows; patterns draw from another alphabet so that a text holds a pattern only where it is put
ROW_ALPHABET = (b"a", b"b") + CP_BYTES
PATTERN_ALPHABET = (b"c", b"d", b"e") + CP_BYTES
BINARY_EXTRA = (b"\x00", b"\xff", b"\x80")
TYPES = {"string": pa.string(), "large_string": pa.large_string(), "binary": pa.binary(), "large_binary": pa.large_binary()}
UTF8_TYPES = (pa.string(), pa.large_string())


def text(rng, n: int, utf8: bool, alphabet=ROW_ALPHABET) -> bytes:
    """exactly n bytes of whole code points drawn from alphabet, padded with its first byte; binary text also draws NUL,
    0x80 and 0xff"""
    pieces = alphabet + (() if utf8 else BINARY_EXTRA)
    idx = rng.integers(len(pieces), size=n)
    ends = np.cumsum(np.array([len(x) for x in pieces])[idx])
    k = int(np.searchsorted(ends, n, side="right"))  # the pieces that fit whole
    head = b"".join([pieces[i] for i in idx[:k].tolist()])
    return head + alphabet[0][:1] * (n - len(head))


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
# (a, b, k): a and b have the same length and first differ at byte k; every pair is whole code points, so it can stand
# at a code point boundary of a utf8 row and keep it valid.  ASCII, NUL and DEL; lead bytes of 2 and 4 byte code points
# (unsigned order: 0xc2 < 0xdf, 0xf0 < 0xf4); continuation bytes at positions 1, 2 and 3.
DIFF_PIECES = ((b"x", b"y", 0), (b"\x00", b"\x7f", 0), ("\u0080".encode(), "\u07ff".encode(), 0),
               ("\u00e9".encode(), "\u00ea".encode(), 1), ("\u0800".encode(), "\u0801".encode(), 2),
               ("\U00010000".encode(), "\U0010ffff".encode(), 0), ("\U00010000".encode(), "\U00010001".encode(), 3))
BINARY_DIFF_PIECES = ((b"\x80", b"\x7f", 0), (b"\xff", b"\x00", 0))


def boundary(row: bytes, p: int) -> int:
    """the last code point boundary at or before byte p of a valid UTF-8 row"""
    while 0 < p < len(row) and (row[p] & 0xC0) == 0x80:
        p -= 1
    return p


# Byte pairs (d1, d2) that share a 256-byte step of warp_first_diff (32 lanes of 8 bytes): lanes 1 and 31 of step 0,
# 5 and 30 of step 1, 0 and 9 of step 4, 1 and 4 of step 8; (1032, 1036) share one 8-byte word.  A variant changes both
# bytes, in opposite directions, so only the lowest difference gives the right order.
MULTI_DIFF = ((10, 250), (300, 500), (1030, 1100), (1032, 1036), (2060, 2080))


def compare_family(rng, length: int, utf8: bool):
    """(base, variants): a base row of `length` bytes and rows around it -- itself; rows of the same length that first
    differ from it at byte d, for every d in DIFF_AT and length - 1 (a bigger byte at some, a smaller one at others);
    rows differing at both bytes of a MULTI_DIFF pair, the first bigger and the second smaller and the reverse; proper
    prefixes of 0, 1, 7, 8 and 9 bytes and one a code point short; the base extended by a byte, by a 4-byte code point,
    by one NUL and by two"""
    pieces = DIFF_PIECES + (() if utf8 else BINARY_DIFF_PIECES)
    pairs = [(d1, d2) for d1, d2 in MULTI_DIFF if d2 < length]
    multi = {d for pair in pairs for d in pair}  # these bytes are "m" in the base: "n" is bigger, "l" smaller
    cuts = sorted({d for d in DIFF_AT + (length - 1,) if 0 <= d < length} | multi)
    parts, plan, pos = [], [], 0  # plan: (byte where the piece starts, the base's piece, the variant's piece)
    for j, d in enumerate(cuts):
        a, b, k = pieces[(j + length) % len(pieces)]
        nxt = cuts[j + 1] if j + 1 < len(cuts) else length
        if d in multi:
            a, b, k = b"m", b"n", 0
        elif d - k < pos or d - k + len(a) > nxt:  # the piece would overlap its neighbour: one ASCII byte instead
            a, b, k = b"x", b"y", 0
        if j % 2 and d not in multi:
            a, b = b, a
        parts += [text(rng, d - k - pos, utf8), a]
        plan.append((d - k, a, b))
        pos = d - k + len(a)
    parts.append(text(rng, length - pos, utf8))
    base = b"".join(parts)
    assert len(base) == length
    variants = [base] + [base[:at] + b + base[at + len(a):] for at, a, b in plan]
    for d1, d2 in pairs:
        for first, second in ((b"n", b"l"), (b"l", b"n")):
            variants.append(base[:d1] + first + base[d1 + 1:d2] + second + base[d2 + 1:])
    for p in (0, 1, 7, 8, 9, length - 1):
        if 0 <= p < length:
            variants.append(base[:boundary(base, p) if utf8 else p])
    variants += [base + b"a", base + "\U0010ffff".encode(), base + b"\x00", base + b"\x00\x00"]
    return base, list(dict.fromkeys(variants))


def compare_families(seed: int, utf8: bool, lengths=ROW_LENGTHS + (MIB,)):
    rng = np.random.default_rng(seed)
    return [compare_family(rng, n, utf8) for n in lengths]


# ---------------------------------------------------------------------------------------------------------------------
# substring, prefix and suffix matches
# ---------------------------------------------------------------------------------------------------------------------
def pattern(rng, m: int, utf8: bool) -> bytes:
    """m bytes whose first is c, d or e, which no filler row holds"""
    return b"cde"[rng.integers(3):][:1] + text(rng, m - 1, utf8, PATTERN_ALPHABET)


def classified_like(p: bytes):
    """the LIKE patterns MatchLike::Exec runs as a substring, prefix and suffix match of p"""
    return [b"%" + p + b"%", p + b"%", b"%" + p]


def window_starts(m: int, n_starts: int):
    """every start around a boundary between two lanes' windows of warp_find_in (and between two 32-window steps):
    64 j - m + {0, 1, 2} and 64 j + {-1, 0, 1}, for the boundaries below n_starts"""
    out = set()
    for j in (1, 2, 3, 31, 32, 33, 64, 65):
        for s in (WINDOW * j - m, WINDOW * j - m + 1, WINDOW * j - m + 2, WINDOW * j - 1, WINDOW * j, WINDOW * j + 1):
            if 0 <= s < n_starts:
                out.add(s)
    return sorted(out)


def substring_texts(rng, pat: bytes, utf8: bool):
    """rows for match_substring of pat (m bytes), each holding at most one occurrence:
      * a row of 64 * 66 + m bytes (warp path) with the occurrence at each start of window_starts;
      * rows of m, m + 1, m + 7, m + 8, m + 9, 1023, 1024, 1025, 2049 bytes (both paths) with it at the first and at the
        last possible start, and the same rows cut a byte short, so the occurrence stops one byte early;
      * the pattern with its last byte changed, at the last start, so only the tail fails."""
    m = len(pat)
    rows = []
    filler = lambda n: text(rng, n, utf8)  # noqa: E731  never holds c, d or e, the pattern's first byte
    n = WINDOW * 66 + m
    for s in window_starts(m, n - m + 1):
        rows.append(filler(s) + pat + filler(n - s - m))
    for n in sorted({n for n in (m, m + 1, m + 7, m + 8, m + 9, 1023, 1024, 1025, 2049) if n >= m}):
        first = pat + filler(n - m)
        last = filler(n - m) + pat
        rows += [first, last, last[:boundary(last, n - 1)], first[1:], filler(n - m) + tail_changed(pat)]
    return rows


def tail_changed(pat: bytes) -> bytes:
    """pat with its last byte changed (an ASCII byte to another pattern letter, the last byte of a multi-byte code point
    to another continuation byte, which keeps UTF-8 valid)"""
    last = pat[-1]
    if last >= 0x80:
        return pat[:-1] + bytes([last ^ 1])
    return pat[:-1] + (b"d" if last == ord("c") else b"c")


def self_overlap_cases():
    """(pattern, rows): patterns that overlap themselves, so a search that skips past a partial match misses them"""
    cases = [(b"aab", [b"aaab", b"aab", b"aaaab", b"aa", b"abaab", b"aaa"]),
             (b"abab" * 3 + b"abc", [b"ab" * k + b"c" for k in (5, 6, 7, 8, 40, 600, 1100)] +
              [b"ab" * 1100, b"ab" * 7 + b"ac"])]
    for m in (9, 17, 64, 65):
        p = b"a" * (m - 1) + b"b"
        cases.append((p, [b"a" * k + b"b" for k in (m - 2, m - 1, m, 2 * m, 1100, 2100)] + [b"a" * 3000]))
    return cases


def head_decoy_cases():
    """(pattern, rows): patterns longer than 8 bytes whose first 8 bytes occur many times in a row while the rest never
    matches (find_in's head hits are verified past byte 8), beside rows where the last copy completes it"""
    cases = []
    for m in (9, 15, 16, 17, 33, 66, 100, 1025, 2000):
        head = b"HEADhead"
        tail = (b"t" * (m - 9)) + b"Z"
        p = head + tail
        decoy = head + tail[:-1] + b"Y"
        rows = []
        for copies in (1, 2, 5, 40, 300):
            rows.append(decoy * copies)
            rows.append(decoy * copies + p)
            rows.append((head * copies) + tail[:-1])
        rows.append(head * 400)
        cases.append((p, rows))
    return cases


def affix_rows(rng, pat: bytes, utf8: bool):
    """rows for starts_with / ends_with of pat: pat alone, pat with text after / before it, pat a byte short, pat with
    one byte changed at each of DIFF_AT and m - 1 (ASCII positions only over utf8), and rows shorter than pat"""
    m = len(pat)
    rows = [pat, pat + text(rng, 5, utf8), text(rng, 5, utf8) + pat, pat[:boundary(pat, m - 1)], pat[1:], b"",
            text(rng, 3, utf8)]
    for tail in (1, 600, 1100):
        rows += [pat + text(rng, tail, utf8), text(rng, tail, utf8) + pat]
    for d in sorted({d for d in DIFF_AT + (m - 1,) if 0 <= d < m}):
        if pat[d] < 0x80:
            bad = pat[:d] + (b"e" if pat[d:d + 1] != b"e" else b"c") + pat[d + 1:]
            rows += [bad, bad + text(rng, 2, utf8), text(rng, 2, utf8) + bad]
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# match_like's general matcher
# ---------------------------------------------------------------------------------------------------------------------
# patterns no classifying regex takes: `_`, several `%`, `_` beside 3- and 4-byte code points, `_` last
GENERAL_PATTERNS = ("a_%b__%c", "%a%%b%%%c%", "_%_", "%_", "%a_", "a%_\uffff%_", "%_\U00010000_%",
                    "\U0010ffff_%", "%\u0800__", "_\u07ff%\u0080_", "a%b%c%d%e", "%%_%%b_")


def instantiate(rng, pat: str, size: int, utf8: bool) -> bytes:
    """a row the LIKE pattern matches (up to escapes, which GENERAL_PATTERNS do not use): each `_` one code point (one
    byte over binary) and each `%` filler, sized so the row has about `size` bytes"""
    n_pct = pat.count("%")
    fixed = len(pat.replace("%", "").encode())
    each = max(size - fixed, 0) // max(n_pct, 1)
    out = []
    for ch in pat:
        if ch == "%":
            out.append(text(rng, each, utf8))
        elif ch == "_":
            pick = ROW_ALPHABET if utf8 else ROW_ALPHABET[:2] + BINARY_EXTRA
            out.append(pick[rng.integers(len(pick))])
        else:
            out.append(ch.encode())
    return b"".join(out)


def like_rows(rng, pat: str, utf8: bool):
    """rows on both sides of 1024 bytes for a general LIKE pattern: instances of it, instances with one byte or one code
    point changed, with a code point added or dropped, and rows that end in a 3- or 4-byte code point"""
    rows = []
    for size in (0, 5, 40, 1000, 1020, 1023, 1024, 1025, 1030, 2049):
        r = instantiate(rng, pat, size, utf8)
        rows.append(r)
        rows.append(r + "\uffff".encode())
        rows.append(r + "\U0010ffff".encode())
        rows.append(r[:-1] + b"q" if r and r[-1] < 0x80 else r + b"q")
        rows.append(b"q" + r)
        rows.append(r[1:] if r and r[0] < 0x80 else r)
    rows += [b"", "\U0010ffff".encode(), "\uffff".encode(), b"a\xf4\x8f\xbf\xbf" if utf8 else b"a\xf4", b"a" * 1500]
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# warp layouts
# ---------------------------------------------------------------------------------------------------------------------
def warp_layout(rng):
    """(is_long, null) masks for 32-row groups holding 0, 1, 2, 31 and 32 long rows at random lanes, one with long rows
    at lanes 0 and 31, one with long rows under null slots (and short ones too), and a last, partial group of 13 rows
    whose last row is long"""
    groups = []
    for k in (0, 1, 2, 31, 32):
        g = np.zeros(32, bool)
        g[rng.choice(32, k, replace=False)] = True
        groups.append((g, rng.random(32) < 0.1))
    g = np.zeros(32, bool)
    g[[0, 31]] = True
    groups.append((g, np.zeros(32, bool)))
    g = np.zeros(32, bool)
    g[[0, 5, 6, 17, 31]] = True
    nul = np.zeros(32, bool)
    nul[[0, 6, 17, 20, 31]] = True
    groups.append((g, nul))
    g = np.zeros(13, bool)
    g[[3, 12]] = True
    groups.append((g, np.zeros(13, bool)))
    return np.concatenate([g for g, _ in groups]), np.concatenate([n for _, n in groups])


def layout_compare_rows(rng, is_long, utf8: bool):
    """(left, right) rows for a warp layout: a long slot holds equal-length rows of 1025-2049 bytes (equal, or differing
    at one byte) or rows of which the shorter has more than 1024 bytes; a short slot the same at 0-16 bytes"""
    left, right = [], []
    for lng in is_long:
        n = int(rng.integers(1025, 2050)) if lng else int(rng.integers(0, 17))
        a = text(rng, n, utf8, (b"a", b"b"))
        kind = rng.integers(3)
        if kind == 0:
            b = a
        elif kind == 1 and n:
            d = int(rng.integers(n))
            b = a[:d] + (b"b" if a[d:d + 1] == b"a" else b"a") + a[d + 1:]
        else:
            b = a + text(rng, int(rng.integers(1, 9)), utf8)
        left.append(a)
        right.append(b)
    return left, right


def layout_match_rows(rng, is_long, pat: bytes, utf8: bool):
    """rows for a warp layout and a pattern: a long slot holds more than max(1024, m) bytes, a short one fewer than
    min(64, m) + 64; each holds pat at its start, at its end, in its middle, or nowhere"""
    m, rows = len(pat), []
    for lng in is_long:
        n = int(rng.integers(max(1025, m + 1), max(2050, m + 1026))) if lng else int(rng.integers(0, min(64, m) + 64))
        where = rng.integers(4) if n >= m else 3
        t = text(rng, n - m if where < 3 else n, utf8)
        if where == 0:
            t = pat + t
        elif where == 1:
            t = t + pat
        elif where == 2:
            cut = boundary(t, int(rng.integers(len(t) + 1))) if utf8 else int(rng.integers(len(t) + 1))
            t = t[:cut] + pat + t[cut:]
        rows.append(t)
    return rows


def array(rows, t: pa.DataType, null=None) -> pa.Array:
    """rows (bytes) as an array of type t; utf8 rows must be valid UTF-8"""
    if t in UTF8_TYPES:
        rows = [r.decode("utf-8") for r in rows]
    return pa.array(rows, t, mask=None if null is None else np.asarray(null, bool))


# ---------------------------------------------------------------------------------------------------------------------
# set lookup
# ---------------------------------------------------------------------------------------------------------------------
def set_lookup_strings(rng, utf8: bool):
    """(value set, probes): for a base string of every length 0-40, 1023-1025 and 1 MiB, its variants -- the base with
    one byte changed at 8k - 1, 8k or the last byte, and with one and with two trailing NULs; the value set holds every
    other variant, the probes all of them, so each hit has neighbours that must miss"""
    in_set, probes = [], []
    for n in list(range(41)) + [1023, 1024, 1025, MIB]:
        base = text(rng, n, utf8, (b"a", b"b"))  # ASCII: any byte may change
        fam = [base]
        for d in (7, 8, 15, 16, 1015, 1016, n - 1):
            if 0 <= d < n:
                fam.append(base[:d] + (b"c" if base[d:d + 1] != b"c" else b"d") + base[d + 1:])
        fam += [base + b"\x00", base + b"\x00\x00"]
        fam = list(dict.fromkeys(fam))
        in_set += fam[::2]
        probes += fam
    return in_set, probes


def upload(ctx, arr: pa.Array, align: int = 1):
    """DeviceArray.from_arrow, with the character data placed at device address 8k + align (odd by default)"""
    from arrow_b200 import DeviceArray, DeviceBuffer  # the device library: only device tests call this
    d = DeviceArray.from_arrow(arr, ctx)
    if arr.buffers()[2] is not None and arr.buffers()[2].size > 0:
        host = arr.buffers()[2].to_pybytes()
        buf = ctx.alloc(len(host) + 16)  # room for the aligned word that holds the last byte
        assert buf.ptr % 8 == 0
        ctx.h2d(buf.ptr + align, pa.py_buffer(host).address, len(host))
        ctx.sync()
        d.buffers[2] = DeviceBuffer(ctx, buf.ptr + align, 0, False, keepalive=buf)
    return d
