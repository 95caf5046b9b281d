"""The host restatement of the string transforms (tests/string_transform_ref.py) against the reference's own expected
outputs (tests/golden/kat_string_transform.json) and against pyarrow.compute: random strings of ASCII, 2-, 3- and
4-byte code points, empty rows and nulls for every type; a grid of SliceOptions; every JoinOptions mode over 1-4
operands with array, scalar and null-scalar operands; invalid UTF-8; and the two places where the device and
pyarrow 24 differ on purpose."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import string_transform_ref as R

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_string_transform.json"), encoding="utf-8"))
ALPHABET = ["a", "b", "Z", " ", "é", "ö", "€", "ḍ", "😀", "𝑓"]
MAX, MIN = R.INT64_MAX, R.INT64_MIN
GRID = list(range(-7, 8)) + [1 << 62, -(1 << 62), MIN, MAX]
STEPS = [1, -1, 2, -2, 3, -3, 1 << 62, -(1 << 62)]


def random_strings(n, seed, type_, max_len=12, null_p=0.15):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
            continue
        k = int(rng.integers(0, max_len + 1))
        s = "".join(ALPHABET[i] for i in rng.integers(0, len(ALPHABET), k))
        out.append(s if type_ in R.UTF8_TYPES else s.encode())
    return pa.array(out, type_)


def _arr(vals, type_):
    if type_ in R.UTF8_TYPES:
        return pa.array(vals, type_)
    return pa.array([None if v is None else v.encode() for v in vals], type_)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's expected outputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_kat_lengths_and_case(type_):
    for c in KAT["length"]:
        if c["function"] == "utf8_length" and type_ not in R.UTF8_TYPES:
            continue
        vals = c["input"] if "input" in c else None
        arr = _arr(vals, type_) if vals is not None else pa.array([bytes.fromhex(h) for h in c["input_hex"]],
                                                                  pa.large_binary() if "large" in str(type_) else pa.binary()).view(type_)
        fn = R.binary_length if c["function"] == "binary_length" else R.utf8_length
        out = pa.int64() if type_ in (pa.large_string(), pa.large_binary()) else pa.int32()
        assert fn(arr).equals(pa.array(c["expected"], out)), c
    if type_ in R.UTF8_TYPES:
        for c in KAT["case"]:
            got = R.ascii_case(_arr(c["input"], type_), c["function"] == "ascii_upper")
            assert got.equals(_arr(c["expected"], type_)), c


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_kat_slices(type_):
    utf8 = type_ in R.UTF8_TYPES
    n = 0
    for c in KAT["slice"]:
        if (c["function"] == "utf8_slice_codeunits") != utf8:
            continue
        fn = R.utf8_slice_codeunits if utf8 else R.binary_slice
        assert fn(_arr(c["input"], type_), c["start"], c["stop"], c["step"]).equals(_arr(c["expected"], type_)), c
        n += 1
    assert n >= 18


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_kat_join(type_):
    for c in KAT["join"]:
        ops = [_arr(o["array"], type_) if "array" in o else
               pa.scalar(None if o["scalar"] is None else (o["scalar"] if type_ in R.UTF8_TYPES else o["scalar"].encode()), type_)
               for o in c["operands"]]
        got = R.binary_join_element_wise(ops, type_, c["null_handling"], c["null_replacement"])
        assert got.equals(_arr(c["expected"], type_)), c


# ---------------------------------------------------------------------------------------------------------------------
# against pyarrow.compute
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_random_lengths_and_case(type_):
    for seed in range(4):
        arr = random_strings(500, seed, type_)
        assert R.binary_length(arr).equals(pc.binary_length(arr))
        if type_ in R.UTF8_TYPES:
            assert R.utf8_length(arr).equals(pc.utf8_length(arr))
            assert R.ascii_case(arr, True).equals(pc.ascii_upper(arr))
            assert R.ascii_case(arr, False).equals(pc.ascii_lower(arr))


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_random_slices(type_):
    utf8 = type_ in R.UTF8_TYPES
    fn = R.utf8_slice_codeunits if utf8 else R.binary_slice
    pfn = pc.utf8_slice_codeunits if utf8 else pc.binary_slice
    for seed in range(3):
        arr = random_strings(300, 10 + seed, type_)
        for start, stop, step in [(0, 3, 1), (1, 8, 1), (-4, MAX, 1), (2, -2, 1), (-5, -1, 2), (0, MAX, 3), (-1, MIN, -1),
                                  (6, 0, -2), (-2, -9, -3), (0, 0, 1)]:
            want = fn(arr, start, stop, step)
            nbytes = sum(len(v) for v in R.values(arr) if v is not None)
            out_bytes = sum(len(v) for v in R.values(want) if v is not None)
            if not R.reference_slice_defined(utf8, len(arr), nbytes, start, stop, step, out_bytes):
                continue
            try:
                got = pfn(arr, start, stop, step)
            except pa.ArrowInvalid as e:
                assert "Negative buffer resize" in str(e)
                continue
            assert want.equals(got), (start, stop, step)


@pytest.mark.parametrize("utf8", [True, False], ids=["utf8", "binary"])
@pytest.mark.parametrize("step", STEPS)
def test_slice_option_grid(utf8, step):
    """start and stop over -7..7, +-2^62, INT64_MIN / MAX: equal to pyarrow wherever pyarrow answers; where its output
    estimate wraps negative it raises, and the restatement (like the device) still slices"""
    vals = ["", "a", "ab", "héllo", "𝑓öõḍšx", None, "abcdefghij"]
    arr = pa.array(vals, pa.string()) if utf8 else pa.array([None if v is None else v.encode() for v in vals], pa.binary())
    fn = R.utf8_slice_codeunits if utf8 else R.binary_slice
    pfn = pc.utf8_slice_codeunits if utf8 else pc.binary_slice
    nbytes = sum(len(v) for v in R.values(arr) if v is not None)
    compared = raised = 0
    for start in GRID:
        for stop in GRID:
            want = fn(arr, start, stop, step)
            assert len(want) == len(arr) and want.null_count == 1
            out_bytes = sum(len(v) for v in R.values(want) if v is not None)
            if not R.reference_slice_defined(utf8, len(arr), nbytes, start, stop, step, out_bytes):
                continue
            try:
                got = pfn(arr, start, stop, step)
            except pa.ArrowInvalid as e:
                assert "Negative buffer resize" in str(e)
                assert R.reference_max_codeunits(utf8, len(arr), nbytes, start, stop, step) < 0
                raised += 1
                continue
            assert want.equals(got), (start, stop, step)
            compared += 1
    # binary_slice with a step below -2^31 is never safe to call in pyarrow: the restatement stands alone there
    assert compared >= (0 if not utf8 and step < -(1 << 31) else 250), compared


def test_slice_step_zero_and_missing_options():
    arr = pa.array(["abc"])
    for fn in (R.utf8_slice_codeunits, R.binary_slice):
        with pytest.raises(ValueError, match="Slice step cannot be zero"):
            fn(arr, 0, 1, 0)
    with pytest.raises(pa.ArrowInvalid, match="Slice step cannot be zero"):
        pc.utf8_slice_codeunits(arr, 0, 1, 0)


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
@pytest.mark.parametrize("mode", R.NULL_HANDLING)
def test_join_modes(type_, mode):
    rng = np.random.default_rng(7)
    utf8 = type_ in R.UTF8_TYPES
    enc = (lambda s: s) if utf8 else (lambda s: s.encode())
    arrays = [random_strings(200, 30 + k, type_, max_len=5, null_p=0.2) for k in range(5)]
    scalars = [pa.scalar(enc("xy"), type_), pa.scalar(enc(""), type_), pa.scalar(None, type_), pa.scalar(enc("é€"), type_)]
    for n_ops in range(1, 5):
        for trial in range(12):
            ops = []
            for k in range(n_ops):
                if rng.random() < 0.3 and k > 0:
                    ops.append(scalars[int(rng.integers(0, len(scalars)))])
                else:
                    ops.append(arrays[int(rng.integers(0, len(arrays)))])
            if not any(isinstance(o, pa.Array) for o in ops):
                ops[0] = arrays[0]
            repl = "NULL" if trial % 2 else ""
            if mode == "skip":  # pyarrow drops the rows whose values are all null (see the divergence test): keep them out
                cols = [R.values(o) if isinstance(o, pa.Array) else [o.as_py()] * 200 for o in ops[:-1]]
                keep = pa.array([n_ops == 1 or any(c[i] is not None for c in cols) for i in range(200)])
                ops = [o.filter(keep) if isinstance(o, pa.Array) else o for o in ops]
            want = R.binary_join_element_wise(ops, type_, mode, repl)
            got = pc.binary_join_element_wise(*ops, null_handling=mode, null_replacement=repl)
            assert want.equals(got), (n_ops, trial)


# ---------------------------------------------------------------------------------------------------------------------
# invalid UTF-8 and the divergences
# ---------------------------------------------------------------------------------------------------------------------
INVALID_UTF8 = [  # (case, rows): both the restatement and pyarrow raise for every slice that walks the bad bytes
    ("stray continuation", [b"a\x80bc"]),
    ("invalid lead byte", [b"a\xffbc"]),
    ("sequence truncated mid-row", [b"a\xe2\x82bc"]),
    ("lead byte at the last row's end", [b"ab\xe2"]),
]
INVALID_SLICES = [(0, 10, 1), (1, 10, 1), (0, 10, 2), (-1, -10, -1), (-10, 10, 1), (0, 3, 1), (-1, MAX, 1)]


def _with_nulls(rows, valid, type_=pa.string()):
    data, offs = b"".join(rows), np.cumsum([0] + [len(r) for r in rows]).astype(np.int32)
    return pa.Array.from_buffers(type_, len(rows), [pa.array(valid).buffers()[1], pa.py_buffer(offs.tobytes()),
                                                    pa.py_buffer(data)], null_count=valid.count(False))


@pytest.mark.parametrize("case,rows", INVALID_UTF8, ids=[c for c, _ in INVALID_UTF8])
def test_invalid_utf8_table(case, rows):
    arr = pa.array(rows, pa.binary()).view(pa.string())
    for sl in INVALID_SLICES:
        with pytest.raises(R.InvalidUtf8):
            R.utf8_slice_codeunits(arr, *sl)
        with pytest.raises(pa.ArrowInvalid, match=R.INVALID_UTF8):
            pc.utf8_slice_codeunits(arr, *sl)
    # a slice that stops before the bad bytes: both fail, or both give the same result, since both decode the code
    # point at `stop` too
    for sl in [(0, 1, 1), (0, 0, 1), (-1, -1, 1), (3, 1, 1)]:
        try:
            want = R.utf8_slice_codeunits(arr, *sl)
        except R.InvalidUtf8:
            with pytest.raises(pa.ArrowInvalid, match=R.INVALID_UTF8):
                pc.utf8_slice_codeunits(arr, *sl)
        else:
            assert want.equals(pc.utf8_slice_codeunits(arr, *sl)), sl
    # a null row is never walked
    nulled = _with_nulls(rows + [b"ok"], [False] * len(rows) + [True])
    assert R.utf8_slice_codeunits(nulled, 0, 10).equals(pc.utf8_slice_codeunits(nulled, 0, 10))


def test_invalid_utf8_across_rows_divergence():
    """A sequence cut off by its row's end (or, backwards, its start): the reference's decoder reads on into the
    neighbouring row and succeeds when those bytes complete it; the restatement and the device stay inside the row and
    raise."""
    lead_at_end = _with_nulls([b"ab\xe2", b"\x82\xacz"], [True, False])
    assert pc.utf8_slice_codeunits(lead_at_end, 0, 10).view(pa.binary()).to_pylist() == [b"ab\xe2", None]
    assert pc.utf8_slice_codeunits(lead_at_end, 0, 10, 2).view(pa.binary()).to_pylist() == [b"a\xe2\x82\xac", None]
    cont_at_start = _with_nulls([b"z\xe2\x82", b"\xacab"], [False, True])
    assert pc.utf8_slice_codeunits(cont_at_start, -1, -10, -1).view(pa.binary()).to_pylist() == [None, b"ba\xe2\x82\xac"]
    for arr, sl in [(lead_at_end, (0, 10, 1)), (lead_at_end, (0, 10, 2)), (cont_at_start, (-1, -10, -1))]:
        with pytest.raises(R.InvalidUtf8):
            R.utf8_slice_codeunits(arr, *sl)


@pytest.mark.parametrize("type_", R.BINARY_TYPES, ids=str)
def test_binary_slice_default_stop_divergence(type_):
    """pyarrow 24's binary_slice estimates its output as n_rows * (stop - start) in int64 without clamping, so the
    default stop overflows it on any array of two or more rows; the device sizes its output from each row and slices"""
    arr = pa.array([b"abc", b"de", None, b"fghij"], type_)
    with pytest.raises(pa.ArrowInvalid, match="Negative buffer resize: -"):
        pc.binary_slice(arr, start=1)
    assert R.binary_slice(arr, 1).to_pylist() == [b"bc", b"e", None, b"ghij"]
    assert pc.binary_slice(arr[:1], start=1).to_pylist() == [b"bc"]  # one row: no overflow
    # utf8_slice_codeunits clamps stop to the input's size and has no such defect
    s = pa.array(["abc", "de", None, "fghij"])
    assert pc.utf8_slice_codeunits(s, start=1).equals(R.utf8_slice_codeunits(s, 1))


@pytest.mark.parametrize("type_", R.BINARY_LIKE, ids=str)
def test_join_skip_all_null_row_divergence(type_):
    """Under SKIP a row whose values are all null (its separator valid) joins nothing, and pyarrow 24 appends no row
    for it at all, so its output is shorter than its input; the restatement and the device give that row ""."""
    enc = (lambda s: s) if type_ in R.UTF8_TYPES else (lambda s: s.encode())
    a = pa.array([None, enc("a"), None], type_)
    b = pa.array([None, enc("b"), None], type_)
    got = pc.binary_join_element_wise(a, b, pa.scalar(enc("-"), type_), null_handling="skip")
    assert got.to_pylist() == [enc("a-b")]
    want = R.binary_join_element_wise([a, b, pa.scalar(enc("-"), type_)], type_, "skip")
    assert want.to_pylist() == [enc(""), enc("a-b"), enc("")]


def test_join_int32_capacity_message():
    """over int32 offsets the join's output is capped at 2^31 - 2 bytes (BaseBinaryBuilder::ReserveData)"""
    big = pa.py_buffer(b"x" * ((1 << 30) - 1))
    scalar = pa.Array.from_buffers(pa.binary(), 1, [None, pa.py_buffer(np.array([0, (1 << 30) - 1], np.int32).tobytes()), big])[0]
    fits = pa.array([b"", b""])            # 2 * (2^30 - 1) = 2^31 - 2 bytes: the limit
    over = pa.array([b"y", b""])           # one byte more
    got = pc.binary_join_element_wise(fits, scalar, b"")
    assert len(got) == 2 and np.frombuffer(got.buffers()[1], np.int32)[-1] == (1 << 31) - 2
    del got
    with pytest.raises(pa.ArrowCapacityError) as e:
        pc.binary_join_element_wise(over, scalar, b"")
    assert str(e.value) == R.join_capacity_error((1 << 31) - 1)


def test_join_null_handling_codes(tmp_path):
    """JOIN_NULL_HANDLING against B2JoinNullHandling as the C compiler sees it and against the reference's
    JoinOptions::NullHandlingBehavior (the integer a serialized pyarrow JoinOptions carries); the B2JoinOperand layout
    against its ctypes mirror"""
    import ctypes as C
    import shutil
    import subprocess

    from arrow_b200 import _cabi as cabi

    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = {k: "B2_JOIN_" + k.upper() for k in cabi.JOIN_NULL_HANDLING}
    lines = [f'printf("{e} %d\\n", (int){e});' for e in names.values()]
    lines.append('printf("size %zu\\n", sizeof(B2JoinOperand));')
    lines += [f'printf("{f} %zu\\n", offsetof(B2JoinOperand, {f}));' for f, _ in cabi.B2JoinOperand._fields_]
    src = tmp_path / "join.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "arrow_b200.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0; }\n")
    exe = tmp_path / "join"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for key, code in cabi.JOIN_NULL_HANDLING.items():
        assert int(got[names[key]]) == code, key
        opts = pa.ipc.open_file(pc.JoinOptions(key).serialize()).read_all().to_pylist()[0][""]
        assert opts["null_handling"] == code, key
    assert int(got["size"]) == C.sizeof(cabi.B2JoinOperand)
    for f, _ in cabi.B2JoinOperand._fields_:
        assert int(got[f]) == getattr(cabi.B2JoinOperand, f).offset, f
