"""String predicates on the device (csrc/string_predicates.cu) against the exact restatement (string_predicates_ref) and
pyarrow.compute, data bits under null slots included: every match function x type, every compare op x shape x type pair
(mixed offset widths, a null scalar), lengths around the 32-row groups, sliced inputs whose offset is not byte-aligned, a
data buffer at an odd address, empty strings and patterns, 1 MiB rows and a 1 MiB scalar on the warp-cooperative path,
the LIKE dispatch, error codes and messages, launches per call and a large_utf8 input of more than 2^32 data bytes."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import string_predicates_ref as ref
from tests.string_boundaries import upload
from tests.test_string_predicates_oracle import TYPES, random_pattern, random_strings

pytestmark = pytest.mark.gpu
COMPARES = tuple(ref.COMPARE)
MATCHES = ("match_substring", "starts_with", "ends_with", "match_like")
LENGTHS = (0, 1, 31, 32, 33, 63, 64, 65, 1000)
PATTERNS = ["", "a", "ab", "%", "%%", "a%", "%a", "%a%", "%ab%", "%a\\b%", "%a\\%", "a\\", "%\\", "_", "a_", "%_%", "a%b",
            "a%b_c%", "%\n%", "é", "_é%", "%é_", "\\%%", "\\____", "(%", "\\\\%", "a.b*", "%[%", "a%%%b"]


def check_match(ctx, function, arr: pa.Array, pattern, pyarrow=True):
    got = getattr(bc, function)(upload(ctx, arr), pattern).to_arrow()
    data, valid = ref.string_match(function, arr, pattern)
    assert got.equals(ref.to_arrow(data, valid)), (function, arr.type, pattern, len(arr))
    np.testing.assert_array_equal(ref.raw_bits(got), data, err_msg=f"{function} {pattern!r} {arr.type}")
    if pyarrow:
        assert got.equals(getattr(pc, function)(arr, pattern))
    return got


def check_compare(ctx, op, left, right):
    """each side: pa.Array (uploaded) or a pa.Scalar"""
    dl = upload(ctx, left) if isinstance(left, pa.Array) else left
    dr = upload(ctx, right) if isinstance(right, pa.Array) else right
    got = getattr(bc, op)(dl, dr).to_arrow()
    rl = left if isinstance(left, pa.Array) else (left.as_buffer().to_pybytes() if left.is_valid else None)
    rr = right if isinstance(right, pa.Array) else (right.as_buffer().to_pybytes() if right.is_valid else None)
    data, valid = ref.compare(op, rl, rr)
    assert got.equals(ref.to_arrow(data, valid)), (op, left.type, right.type)
    np.testing.assert_array_equal(ref.raw_bits(got), data, err_msg=f"{op} {left.type} {right.type}")
    assert got.equals(getattr(pc, op)(left, right))


@pytest.mark.parametrize("tname", list(TYPES))
@pytest.mark.parametrize("function", MATCHES)
def test_match_types_lengths(ctx, tname, function):
    t = TYPES[tname]
    rng = np.random.default_rng(len(tname) * 31 + MATCHES.index(function))
    for n in LENGTHS:
        arr = random_strings(rng, n + 5, t)
        for p in PATTERNS + [random_pattern(rng, t) for _ in range(4)]:
            if function != "match_like" or not (t in ref.UTF8_TYPES and isinstance(p, bytes) and not ref._valid_utf8(p)):
                check_match(ctx, function, arr.slice(0, n), p)
                check_match(ctx, function, arr.slice(5), p)  # offset 5: not byte-aligned


@pytest.mark.parametrize("tname", list(TYPES))
def test_match_edges(ctx, tname):
    t = TYPES[tname]
    enc = (lambda s: s) if t in ref.UTF8_TYPES else (lambda s: s.encode())
    empty = pa.array([enc("")] * 40 + [None, enc("a")], t)
    long_pattern = "x" * 50
    short = pa.array([enc("x" * k) for k in range(49)] + [None], t)
    for f in MATCHES:
        for p in ("", "%", "a", long_pattern):
            check_match(ctx, f, empty, p)
            check_match(ctx, f, short, p)  # a pattern longer than every row
    allnull = pa.array([None] * 70, t)
    for f in MATCHES:
        check_match(ctx, f, allnull, "a")


@pytest.mark.parametrize("lname", list(TYPES))
@pytest.mark.parametrize("rname", list(TYPES))
def test_compare_shapes_type_pairs(ctx, lname, rname):
    lt, rt = TYPES[lname], TYPES[rname]
    rng = np.random.default_rng(7 * len(lname) + len(rname))
    for n in (0, 1, 33, 65, 1000):
        left = random_strings(rng, n + 3, lt, 4).slice(3)
        right = random_strings(rng, n, rt, 4)
        s = ref.slots(right)[0] if n else b"ab"
        sc = pa.scalar(s.decode() if rt in ref.UTF8_TYPES else s, rt)
        for op in COMPARES:
            check_compare(ctx, op, left, right)
            check_compare(ctx, op, left, sc)
            check_compare(ctx, op, sc, left)
            check_compare(ctx, op, left, pa.scalar(None, rt))
            check_compare(ctx, op, pa.scalar(None, rt), left)


def test_compare_bytes_order(ctx):
    """unsigned bytes, a proper prefix first: b"\\xff" > b"a", b"ab" < b"abc" < b"abd" """
    arr = pa.array([b"\xff", b"a", b"", b"ab", b"abc", b"abd", b"\x00", b"a\x00"], pa.binary())
    for op in COMPARES:
        for s in (b"a", b"ab", b"\xff", b"", b"abc\x00"):
            check_compare(ctx, op, arr, pa.scalar(s, pa.binary()))
    assert bc.greater(DeviceArray.from_arrow(pa.array([b"\xff"], pa.binary()), ctx), b"a").to_arrow().to_pylist() == [True]


def test_python_operands(ctx):
    d = DeviceArray.from_arrow(pa.array(["MAIL", "SHIP", None, "AIR"]), ctx)
    assert bc.equal(d, "MAIL").to_arrow().to_pylist() == [True, False, None, False]
    assert bc.less("M", d).to_arrow().to_pylist() == [True, True, None, False]
    assert bc.call_function("greater_equal", [d, pa.scalar("M")]).to_arrow().to_pylist() == [True, True, None, False]
    assert bc.call_function("match_like", [d], pc.MatchSubstringOptions("%AI%")).to_arrow().to_pylist() == [True, False, None, True]
    assert bc.call_function("starts_with", [d], {"pattern": "S"}).to_arrow().to_pylist() == [False, True, None, False]
    for name in MATCHES:
        assert name in bc.list_functions()


def _long_rows(t, row_len, tail):
    body = b"ab" * (row_len // 2)
    rows = [body[: row_len - len(tail)] + tail, body[:row_len], None, b"x", tail]
    if t in ref.UTF8_TYPES:
        rows = [None if r is None else r.decode() for r in rows]
    return pa.array(rows, t)


@pytest.mark.parametrize("tname", list(TYPES))
def test_long_rows(ctx, tname):
    """1 MiB rows take the warp-cooperative path: the match at the very end, and straddling each lane's window and
    each 32-window step"""
    t = TYPES[tname]
    mib = 1 << 20
    for tail in (b"XYZ", b"QRSTUVWXYZ0123456789"):
        arr = _long_rows(t, mib, tail)
        for f in ("match_substring", "ends_with", "match_like"):
            check_match(ctx, f, arr, ("%" if f == "match_like" else "") + tail.decode())
        check_match(ctx, "starts_with", arr, "abab")
    for start in (64 - 1, 64 * 32 - 2, 64 * 32 * 3 - 5, 5000):
        for m in (2, 9, 20):
            raw = bytearray(b"a" * mib)
            raw[start:start + m] = b"Z" * m
            arr = pa.array([bytes(raw), bytes(raw[: start + m - 1])], pa.binary())
            check_match(ctx, "match_substring", arr.cast(t), "Z" * m)
    big = pa.array([b"ab" * (mib // 2) + b"c", b"ab" * (mib // 2), b"ab" * (mib // 2) + b"b", None], pa.binary()).cast(t)
    for op in COMPARES:
        check_compare(ctx, op, big, big)
        check_compare(ctx, op, big, pa.scalar(b"ab" * (mib // 2), pa.binary()).cast(t))  # a 1 MiB scalar
        check_compare(ctx, op, pa.scalar(b"ab" * (mib // 2) + b"b", pa.binary()).cast(t), big)


def test_like_dispatch(ctx):
    """b2_string_match_create classifies LIKE patterns as MatchLike::Exec does"""
    names = {"match_substring": "match_substring", "starts_with": "starts_with", "ends_with": "ends_with", "regex": "match_like"}
    rng = np.random.default_rng(99)
    pats = [p.encode() for p in PATTERNS] + [random_pattern(rng, pa.binary()) for _ in range(300)]
    for utf8 in (True, False):
        for p in pats:
            try:
                kind, lit = ref.like_plan(p, utf8)
            except ref.InvalidPattern:
                with pytest.raises(pa.ArrowInvalid, match="Invalid regular expression: invalid UTF-8"):
                    bc.string_match_plan(p, utf8)
                continue
            runs, nbytes = bc.string_match_plan(p, utf8)
            assert runs == names[kind], (p, utf8)
            if kind != "regex":
                assert nbytes == len(lit), (p, utf8)


def test_errors(ctx):
    d = DeviceArray.from_arrow(pa.array(["a", "b"]), ctx)
    db = DeviceArray.from_arrow(pa.array([b"a", b"b"]), ctx)
    num = DeviceArray.from_arrow(pa.array([1, 2]), ctx)
    for f in MATCHES:
        with pytest.raises(pa.ArrowNotImplementedError, match="ignore_case"):
            getattr(bc, f)(d, "a", ignore_case=True)
        with pytest.raises(pa.ArrowInvalid, match=f"Function '{f}' cannot be called without options"):
            bc.call_function(f, [d])
        with pytest.raises(pa.ArrowNotImplementedError, match=r"has no kernel matching input types \(int64\)"):
            getattr(bc, f)(num, "a")
    with pytest.raises(pa.ArrowInvalid, match="Invalid regular expression: invalid UTF-8"):
        bc.match_like(d, b"%\xa9b%")
    assert bc.match_like(db, b"%\xa9b").to_arrow().to_pylist() == [False, False]
    for op in COMPARES:
        with pytest.raises(pa.ArrowNotImplementedError, match=r"Function '\w+' has no kernel matching input types \(string, int64\)"):
            getattr(bc, op)(d, 1)
        with pytest.raises(pa.ArrowNotImplementedError, match="no kernel matching input types"):
            getattr(bc, op)(d, num)
    # a handle compiled for utf8 refuses binary input, and the reverse
    lib = ctx.lib
    h = C.c_void_p()
    assert lib.b2_string_match_create(ctx.handle, 0, b"a", 1, 1, C.byref(h), ctx.stream) == 0
    try:
        cin, cout = db._c(), _cabi.B2Array()
        assert lib.b2_string_match(h, C.byref(cin), C.byref(cout), ctx.stream) == 3  # B2_TYPE_ERROR
    finally:
        lib.b2_string_match_destroy(h)


def test_launches_per_call(ctx):
    """one kernel per call; one more to re-base the validity of an input with nulls"""
    lib = _cabi.lib()
    for arr, extra in ((pa.array(["a", "ab", "b"] * 100), 0), (pa.array(["a", None, "b"] * 100), 1)):
        d = DeviceArray.from_arrow(arr, ctx)
        for call in (lambda: bc.match_substring(d, "ab"), lambda: bc.match_like(d, "a%b_c%"), lambda: bc.equal(d, "ab"),
                     lambda: bc.less(d, d)):
            before = lib.b2_launch_count()
            call()
            ctx.sync()
            assert lib.b2_launch_count() - before == 1 + extra


def test_more_than_4gib_of_bytes(ctx):
    """a large_utf8 column with more than 2^32 data bytes: equal / starts_with / ends_with counts against torch"""
    torch = pytest.importorskip("torch")
    n = 140_000_000
    g = torch.Generator(device="cuda").manual_seed(11)
    lens = torch.randint(0, 64, (n,), dtype=torch.int64, device="cuda", generator=g)
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offs[1:])
    total = int(offs[-1])
    assert total > (1 << 32)
    data = (torch.randint(0, 2, (total,), dtype=torch.uint8, device="cuda", generator=g) + ord("a"))
    torch.cuda.synchronize()
    d = DeviceArray.from_pointers(ctx, pa.large_string(), n, offs.data_ptr(), data2_ptr=data.data_ptr(), keepalive=(offs, data))
    o0 = offs[:-1]
    ok = lens >= 2
    first = torch.where(ok, data[o0.clamp(max=total - 2)], 0)
    second = torch.where(ok, data[(o0 + 1).clamp(max=total - 1)], 0)
    last = torch.where(ok, data[(offs[1:] - 1).clamp(min=0)], 0)
    penult = torch.where(ok, data[(offs[1:] - 2).clamp(min=0)], 0)
    a, b = ord("a"), ord("b")
    want_eq = int(((lens == 2) & (first == a) & (second == b)).sum())
    want_sw = int((ok & (first == a) & (second == b)).sum())
    want_ew = int((ok & (penult == a) & (last == b)).sum())
    for got, want in ((bc.equal(d, "ab"), want_eq), (bc.starts_with(d, "ab"), want_sw), (bc.ends_with(d, "ab"), want_ew)):
        arr = got.to_arrow()
        assert arr.null_count == 0
        assert pc.sum(arr).as_py() == want
