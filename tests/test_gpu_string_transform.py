"""The device's string transforms (csrc/string_transform.cu) against the host restatement (tests/string_transform_ref.py)
and pyarrow.compute: every function and type over row counts around 32-row groups, slices whose offset is not
byte-aligned over character data at an odd device address, 1 MiB rows, the full SliceOptions grid, every JoinOptions
mode with array, scalar and null-scalar operands, errors and their texts, invalid UTF-8, launches per call, a
large_utf8 input of more than 2^32 bytes, and the int32 join's capacity limit.  Slices and joins must be byte-identical
to the reference's buffers; the lengths and case maps equal as arrays."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import string_transform_ref as R
from tests.string_boundaries import upload
from tests.test_string_transform_oracle import GRID, INVALID_SLICES, INVALID_UTF8, STEPS, _with_nulls, random_strings

pytestmark = pytest.mark.gpu
LENGTHS = (0, 1, 31, 32, 33, 1000)
SLICES = [(0, 3, 1), (1, 8, 1), (-4, R.INT64_MAX, 1), (2, -2, 1), (-5, -1, 2), (0, R.INT64_MAX, 3), (-1, R.INT64_MIN, -1),
          (6, 0, -2), (-2, -9, -3), (0, 0, 1), (0, 8, 1), (-4, R.INT64_MAX, 1)]


def offsets_and_data(arr: pa.Array):
    wide = arr.type in (pa.large_string(), pa.large_binary())
    offs = np.frombuffer(arr.buffers()[1], np.int64 if wide else np.int32, count=arr.offset + len(arr) + 1)[arr.offset:]
    data = arr.buffers()[2].to_pybytes()[int(offs[0]):int(offs[-1])] if arr.buffers()[2] is not None else b""
    return offs, data


def same_buffers(got: pa.Array, want: pa.Array, what=""):
    """equal arrays with identical offsets and character bytes (null slots included)"""
    assert got.equals(want), what
    go, gd = offsets_and_data(got)
    wo, wd = offsets_and_data(want)
    np.testing.assert_array_equal(go - go[0], wo - wo[0], err_msg=str(what))
    assert gd == wd, what


def dev(ctx, arr, cut=3, align=1):
    """arr sliced at `cut` (an offset that is not byte-aligned) with its characters at an odd device address"""
    return upload(ctx, arr, align).slice(cut, len(arr) - cut) if cut else upload(ctx, arr, align)


def _slice_fn(utf8):
    return (bc.utf8_slice_codeunits, R.utf8_slice_codeunits, pc.utf8_slice_codeunits) if utf8 else \
           (bc.binary_slice, R.binary_slice, pc.binary_slice)


def check_slice(ctx, arr: pa.Array, start, stop, step, darr=None):
    utf8 = arr.type in R.UTF8_TYPES
    fn, rfn, pfn = _slice_fn(utf8)
    got = fn(darr if darr is not None else upload(ctx, arr), start, stop, step).to_arrow()
    want = rfn(arr, start, stop, step)
    same_buffers(got, want, (arr.type, start, stop, step))
    nbytes = sum(len(v) for v in R.values(arr) if v is not None)
    out_bytes = sum(len(v) for v in R.values(want) if v is not None)
    if R.reference_slice_defined(utf8, len(arr), nbytes, start, stop, step, out_bytes):
        try:
            same_buffers(got, pfn(arr, start, stop, step), ("pyarrow", arr.type, start, stop, step))
        except pa.ArrowInvalid as e:
            assert "Negative buffer resize" in str(e)
    return got


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_lengths_and_case(ctx, type_):
    for n in LENGTHS:
        arr = random_strings(n + 3, 100 + n, type_)
        d = dev(ctx, arr)
        host = arr.slice(3)
        got = bc.binary_length(d).to_arrow()
        assert got.equals(R.binary_length(host)) and got.equals(pc.binary_length(host)), n
        if type_ in R.UTF8_TYPES:
            got = bc.utf8_length(d).to_arrow()
            assert got.equals(R.utf8_length(host)) and got.equals(pc.utf8_length(host)), n
            for upper, fn in ((True, bc.ascii_upper), (False, bc.ascii_lower)):
                got = fn(d).to_arrow()
                assert got.equals(R.ascii_case(host, upper)), n
                # the reference maps the contiguous span, null slots included, and re-bases the offsets
                same_buffers(got, (pc.ascii_upper if upper else pc.ascii_lower)(host), (n, upper))


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_slices(ctx, type_):
    for n in LENGTHS:
        arr = random_strings(n + 3, 200 + n, type_)
        d = dev(ctx, arr)
        for sl in SLICES:
            check_slice(ctx, arr.slice(3), *sl, darr=d)


@pytest.mark.parametrize("type_", R.UTF8_TYPES, ids=str)
def test_slices_ascii_runs(ctx, type_):
    """rows of ASCII runs 0-20 bytes long between 2-, 3- and 4-byte code points, cut at every length up to 70 bytes, so
    slice bounds fall at every distance from a multi-byte code point"""
    rng = np.random.default_rng(5)
    wide = ["é", "€", "😀"]
    rows = []
    for i in range(1500):
        parts = ["".join(chr(97 + int(c)) for c in rng.integers(0, 26, int(rng.integers(0, 21)))) + wide[int(rng.integers(0, 3))]
                 for _ in range(int(rng.integers(0, 4)))]
        rows.append(None if i % 13 == 0 else "".join(parts)[: int(rng.integers(0, 70))])
    arr = pa.array(rows, type_)
    d = dev(ctx, arr, cut=0, align=5)
    for sl in SLICES + [(3, 17, 1), (-13, -2, 1), (-20, R.INT64_MAX, 1), (9, R.INT64_MAX, 1), (-9, 9, 1), (16, 8, -1),
                        (-17, -30, -2), (8, 40, 5)]:
        check_slice(ctx, arr, *sl, darr=d)


@pytest.mark.parametrize("utf8", [True, False], ids=["utf8", "binary"])
@pytest.mark.parametrize("step", STEPS)
def test_slice_option_grid(ctx, utf8, step):
    vals = ["", "a", "ab", "héllo", "𝑓öõḍšx", None, "abcdefghij"]
    arr = pa.array(vals, pa.large_string()) if utf8 else pa.array([None if v is None else v.encode() for v in vals], pa.binary())
    d = upload(ctx, arr)
    for start in GRID:
        for stop in GRID:
            check_slice(ctx, arr, start, stop, step, darr=d)


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
@pytest.mark.parametrize("mode", R.NULL_HANDLING)
def test_join(ctx, type_, mode):
    rng = np.random.default_rng(11)
    utf8 = type_ in R.UTF8_TYPES
    enc = (lambda s: s) if utf8 else (lambda s: s.encode())
    arrays = [random_strings(n + 3, 300 + k, type_, max_len=5, null_p=0.2).slice(3) for k, n in enumerate((1000, 1000, 1000))]
    devs = [dev(ctx, random_strings(1003, 300 + k, type_, max_len=5, null_p=0.2), align=k + 1) for k in range(3)]
    scalars = [pa.scalar(enc("xy"), type_), pa.scalar(enc(""), type_), pa.scalar(None, type_), pa.scalar(enc("é€"), type_)]
    for n_ops in range(1, 5):
        for trial in range(10):
            pick = [int(rng.integers(0, 3)) if (k == 0 or rng.random() < 0.7) else -1 - int(rng.integers(0, 4))
                    for k in range(n_ops)]
            ops = [arrays[p] if p >= 0 else scalars[-1 - p] for p in pick]
            dops = [devs[p] if p >= 0 else scalars[-1 - p] for p in pick]
            repl = "NUL" if trial % 2 else ""
            got = bc.binary_join_element_wise(*dops, null_handling=mode, null_replacement=repl).to_arrow()
            want = R.binary_join_element_wise(ops, type_, mode, repl)
            same_buffers(got, want, (n_ops, trial))
            if mode != "skip":
                same_buffers(got, pc.binary_join_element_wise(*ops, null_handling=mode, null_replacement=repl))


def test_join_kat_shapes(ctx):
    """separator only, scalar values with an array separator, and SKIP rows whose values are all null"""
    sep = pa.array([None, "-", "--"])
    assert bc.binary_join_element_wise(DeviceArray.from_arrow(sep, ctx)).to_arrow().to_pylist() == [None, "", ""]
    got = bc.binary_join_element_wise("foo", "bar", "", DeviceArray.from_arrow(sep, ctx)).to_arrow()
    assert got.to_pylist() == [None, "foo-bar-", "foo--bar--"]
    a = DeviceArray.from_arrow(pa.array([None, "a", None]), ctx)
    got = bc.binary_join_element_wise(a, a, "-", null_handling="skip").to_arrow()
    assert got.to_pylist() == ["", "a-a", ""]  # pyarrow 24 drops the two all-null rows


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_mib_rows(ctx, type_):
    """1 MiB rows among short ones, so lengths take the warp path, and the slices walk and copy long rows"""
    mib = 1 << 20
    utf8 = type_ in R.UTF8_TYPES
    unit = "aé€😀" if utf8 else "ab\x01"
    long_row = (unit * (mib // len(unit.encode()) + 1)).encode()[:mib]
    if utf8:
        long_row = long_row.decode("utf-8", "ignore").encode()
    rows = [long_row if i % 7 in (0, 3) else b"xy" * (i % 5) for i in range(40)]
    rows[5] = None
    arr = pa.array(rows, pa.large_binary() if "large" in str(type_) else pa.binary()).view(type_)
    d = upload(ctx, arr, 3)
    assert bc.binary_length(d).to_arrow().equals(pc.binary_length(arr))
    if utf8:
        assert bc.utf8_length(d).to_arrow().equals(pc.utf8_length(arr))
        assert bc.ascii_upper(d).to_arrow().equals(pc.ascii_upper(arr))
    for sl in [(0, R.INT64_MAX, 1), (-3, R.INT64_MAX, 1), (5, -5, 1), (1, R.INT64_MAX, 2), (-1, R.INT64_MIN, -1),
               (-2, 10, -3)]:
        check_slice(ctx, arr, *sl, darr=d)


def test_errors(ctx):
    s = DeviceArray.from_arrow(pa.array(["abc", "d"]), ctx)
    b = DeviceArray.from_arrow(pa.array([b"abc", b"d"]), ctx)
    ls = DeviceArray.from_arrow(pa.array(["abc", "d"], pa.large_string()), ctx)
    num = DeviceArray.from_arrow(pa.array([1, 2]), ctx)
    for fn, arg, t in ((bc.utf8_slice_codeunits, s, "string"), (bc.binary_slice, b, "binary")):
        with pytest.raises(pa.ArrowInvalid, match="Slice step cannot be zero"):
            fn(arg, 0, 1, 0)
        with pytest.raises(pa.ArrowInvalid, match=f"Function '{fn.__name__}' cannot be called without options"):
            bc.call_function(fn.__name__, [arg])
    for name, arg, text in (("utf8_slice_codeunits", b, "binary"), ("binary_slice", s, "string"), ("ascii_upper", b, "binary"),
                            ("ascii_lower", num, "int64"), ("utf8_length", b, "binary"), ("binary_length", num, "int64")):
        with pytest.raises(pa.ArrowNotImplementedError, match=rf"Function '{name}' has no kernel matching input types \({text}\)"):
            bc.call_function(name, [arg], {"start": 0} if "slice" in name else None)
    with pytest.raises(pa.ArrowNotImplementedError, match=r"no kernel matching input types \(string, large_string, string\)"):
        bc.binary_join_element_wise(s, ls, "-")
    with pytest.raises(pa.ArrowNotImplementedError, match=r"no kernel matching input types \(string, binary\)"):
        bc.binary_join_element_wise(s, b"-")
    with pytest.raises(ValueError, match="null handling"):
        bc.binary_join_element_wise(s, "-", null_handling="drop")
    # the C ABI's codes
    lib, cout = ctx.lib, _cabi.B2Array()
    assert lib.b2_string_slice(ctx.handle, C.byref(s._c()), 0, 1, 0, 1, C.byref(cout), ctx.stream) == _cabi.INVALID
    assert lib.b2_string_slice(ctx.handle, C.byref(s._c()), 0, 1, 1, 0, C.byref(cout), ctx.stream) == _cabi.NOT_IMPLEMENTED
    assert lib.b2_ascii_case(ctx.handle, C.byref(b._c()), 1, C.byref(cout), ctx.stream) == _cabi.NOT_IMPLEMENTED
    assert lib.b2_string_length(ctx.handle, C.byref(b._c()), 1, C.byref(cout), ctx.stream) == _cabi.NOT_IMPLEMENTED


@pytest.mark.parametrize("case,rows", INVALID_UTF8, ids=[c for c, _ in INVALID_UTF8])
def test_invalid_utf8(ctx, case, rows):
    arr = pa.array(rows, pa.binary()).view(pa.string())
    d = upload(ctx, arr)
    for sl in INVALID_SLICES:
        with pytest.raises(pa.ArrowInvalid, match=R.INVALID_UTF8):
            bc.utf8_slice_codeunits(d, *sl)
    nulled = _with_nulls(rows + [b"ok"], [False] * len(rows) + [True])
    same_buffers(bc.utf8_slice_codeunits(upload(ctx, nulled), 0, 10).to_arrow(), pc.utf8_slice_codeunits(nulled, 0, 10))
    # utf8_length and binary_length validate nothing
    assert bc.utf8_length(d).to_arrow().equals(pc.utf8_length(arr))


def test_invalid_utf8_across_rows(ctx):
    """where the reference's decoder completes a sequence from the neighbouring row, the device raises"""
    lead_at_end = _with_nulls([b"ab\xe2", b"\x82\xacz"], [True, False])
    cont_at_start = _with_nulls([b"z\xe2\x82", b"\xacab"], [False, True])
    for arr, sl in [(lead_at_end, (0, 10, 1)), (lead_at_end, (0, 10, 2)), (cont_at_start, (-1, -10, -1))]:
        pc.utf8_slice_codeunits(arr, *sl)  # the reference succeeds
        with pytest.raises(pa.ArrowInvalid, match=R.INVALID_UTF8):
            bc.utf8_slice_codeunits(upload(ctx, arr), *sl)


def test_binary_slice_default_stop(ctx):
    arr = pa.array([b"abc", b"de", None, b"fghij"] * 9, pa.large_binary())
    got = bc.binary_slice(DeviceArray.from_arrow(arr, ctx), 1).to_arrow()
    same_buffers(got, R.binary_slice(arr, 1))
    with pytest.raises(pa.ArrowInvalid, match="Negative buffer resize"):
        pc.binary_slice(arr, start=1)


def test_call_function_options(ctx):
    """every string transform that takes options, given them as a pyarrow Options object and as a dict"""
    s = DeviceArray.from_arrow(pa.array(["héllo", None, "wörld"]), ctx)
    b = DeviceArray.from_arrow(pa.array([b"hello", None, b"world!"]), ctx)
    cases = {
        "utf8_slice_codeunits": ([s], pc.SliceOptions(1, -1, 2), {"start": 1, "stop": -1, "step": 2},
                                 lambda: bc.utf8_slice_codeunits(s, 1, -1, 2)),
        "binary_slice": ([b], pc.SliceOptions(-5, 4), {"start": -5, "stop": 4}, lambda: bc.binary_slice(b, -5, 4)),
        "binary_join_element_wise": ([s, s, "+"], pc.JoinOptions("replace", "?"), {"null_handling": "replace", "null_replacement": "?"},
                                     lambda: bc.binary_join_element_wise(s, s, "+", null_handling="replace", null_replacement="?")),
    }
    assert set(cases) == set(bc._STRING_TRANSFORM_OPTIONS)
    for name, (args, options, keywords, direct) in cases.items():
        want = direct().to_arrow()
        for o in (options, keywords):
            assert bc.call_function(name, args, o).to_arrow().equals(want), (name, o)
    assert bc.call_function("binary_join_element_wise", [s, s, "+"], pc.JoinOptions("replace", "?")).to_arrow().to_pylist() == \
        ["héllo+héllo", "?+?", "wörld+wörld"]
    for name in ("binary_length", "utf8_length", "ascii_upper", "ascii_lower", *cases):
        assert name in bc.list_functions()


def test_launches_per_call(ctx):
    """lengths and case: one kernel; slices and join: sizes, scan, write; plus one to re-base an input's validity"""
    lib = _cabi.lib()
    for arr, extra in ((pa.array(["ab", "héllo", "c"] * 100), 0), (pa.array(["ab", None, "c"] * 100), 1)):
        d = DeviceArray.from_arrow(arr, ctx)
        b = DeviceArray.from_arrow(arr.cast(pa.binary()), ctx)
        for call, launches in ((lambda: bc.binary_length(d), 1), (lambda: bc.utf8_length(d), 1), (lambda: bc.ascii_upper(d), 1),
                               (lambda: bc.utf8_slice_codeunits(d, 1, 3), 3), (lambda: bc.utf8_slice_codeunits(d, -1, -4, -1), 3),
                               (lambda: bc.binary_slice(b, 1, 5, 2), 3)):
            before = lib.b2_launch_count()
            call()
            ctx.sync()
            assert lib.b2_launch_count() - before == launches + extra
        before = lib.b2_launch_count()
        bc.binary_join_element_wise(d, "x", d, "-", null_handling="replace")
        ctx.sync()
        assert lib.b2_launch_count() - before == 3


def test_more_than_4gib_of_bytes(ctx):
    """a large_utf8 column with more than 2^32 data bytes: lengths, ascii_upper and a slice against torch"""
    torch = pytest.importorskip("torch")
    n = 140_000_000
    g = torch.Generator(device="cuda").manual_seed(12)
    lens = torch.randint(0, 64, (n,), dtype=torch.int64, device="cuda", generator=g)
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offs[1:])
    total = int(offs[-1])
    assert total > (1 << 32)
    data = torch.randint(ord("a"), ord("z") + 1, (total,), dtype=torch.uint8, device="cuda", generator=g)
    torch.cuda.synchronize()
    d = DeviceArray.from_pointers(ctx, pa.large_string(), n, offs.data_ptr(), data2_ptr=data.data_ptr(), keepalive=(offs, data))

    for fn in (bc.binary_length, bc.utf8_length):
        got = fn(d).to_arrow()
        assert got.null_count == 0 and pc.sum(got).as_py() == total
        assert np.array_equal(got.to_numpy()[:1000], lens[:1000].cpu().numpy())
    up = bc.ascii_upper(d)
    head = up.slice(0, 2000).to_arrow()
    want = bytes(data[: int(offs[2000])].cpu().numpy()).upper()
    assert offsets_and_data(head)[1] == want
    tail = up.slice(n - 2000, 2000).to_arrow()
    assert offsets_and_data(tail)[1] == bytes(data[int(offs[n - 2000]):].cpu().numpy()).upper()
    del up
    sl = bc.utf8_slice_codeunits(d, 0, 8)
    got = bc.binary_length(sl).to_arrow()
    assert pc.sum(got).as_py() == int(lens.clamp(max=8).sum())


def test_join_int32_capacity(ctx):
    """over int32 offsets the join may produce 2^31 - 2 bytes and fails past that with the reference's text"""
    big = pa.py_buffer(b"x" * ((1 << 30) - 1))
    scalar = pa.Array.from_buffers(pa.binary(), 1, [None, pa.py_buffer(np.array([0, (1 << 30) - 1], np.int32).tobytes()), big])[0]
    fits = DeviceArray.from_arrow(pa.array([b"", b""]), ctx)
    got = bc.binary_join_element_wise(fits, scalar, b"")
    assert got.length == 2
    lens = bc.binary_length(got).to_arrow().to_pylist()
    assert lens == [(1 << 30) - 1, (1 << 30) - 1]
    del got
    over = DeviceArray.from_arrow(pa.array([b"y", b""]), ctx)
    with pytest.raises(pa.ArrowCapacityError, match=R.join_capacity_error((1 << 31) - 1)):
        bc.binary_join_element_wise(over, scalar, b"")


def test_tile_of_4gib(ctx):
    """the builder stages a 2048-row tile's output offsets in 32 bits: a tile whose output reaches 4 GiB is
    NotImplemented, one just under it is sliced"""
    torch = pytest.importorskip("torch")
    row = 1 << 21
    n = 2048
    offs = torch.arange(0, (n + 1) * row, row, dtype=torch.int64, device="cuda")
    data = torch.full((n * row + 64,), ord("x"), dtype=torch.uint8, device="cuda")
    data[::row] = ord("a")
    torch.cuda.synchronize()
    whole = DeviceArray.from_pointers(ctx, pa.large_binary(), n, offs.data_ptr(), data2_ptr=data.data_ptr(), keepalive=(offs, data))
    with pytest.raises(pa.ArrowNotImplementedError, match="4 GiB or more"):
        bc.binary_slice(whole, 0)
    got = bc.binary_slice(whole.slice(1), 0, R.INT64_MAX)
    lens = bc.binary_length(got).to_arrow()
    assert len(lens) == n - 1 and pc.sum(lens).as_py() == (n - 1) * row
    head = got.slice(0, 2).to_arrow()
    assert head.to_pylist() == [b"a" + b"x" * (row - 1)] * 2
