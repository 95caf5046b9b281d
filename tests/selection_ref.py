"""Exact reference for Filter, Take and the mask -> take-indices conversion, restated row by row and independent of
oracle/arrow_oracle.py.

Rows are held in the form selection moves them, which is never a value:
- a fixed-width row (integers, float16/32/64, temporal types, fixed_size_binary, dictionary indices) is its W raw bytes,
  so NaN payloads, -0.0 and every other bit pattern must come through unchanged;
- a bool row is one bit;
- a binary row (utf8 / binary, 32- or 64-bit offsets) is a Python `bytes`;
- validity is a bool vector.  Null rows carry bytes too, but no comparison looks at them.

Semantics restated from the reference (FilterOptions, compute/api_vector.h:37-51; Take, vector_selection_take_internal.cc and
CheckIndexBounds, util/int_util.cc:452-560):
- Filter DROP keeps the rows whose mask slot is valid and true; EMIT_NULL also keeps the rows whose mask slot is null and
  emits a null there.  Output validity = values validity AND mask validity of the kept rows.
- Take: out[i] = values[idx[i]]; a null index gives a null row and is never checked; the first VALID index outside
  [0, len) raises IndexError("Index <v> out of bounds"), v printed signed for signed index types and unsigned otherwise.
- GetTakeIndices returns uint16 indices for masks of at most 65535 rows and uint32 beyond (vector_selection_take_internal.cc
  :298-305); under EMIT_NULL a null mask slot gives a null index.
- int32-offset capacity (vector_selection_internal.cc:484,519-523): Take fails with "Take operation overflowed binary array
  capacity" as soon as the running output size exceeds kOffsetLimit = 2^31 - 2; Filter has no such check, and needs none:
  its output is never larger than its input, which int32 offsets already keep <= 2^31 - 1 bytes."""
import numpy as np
import pyarrow as pa

from tests.exact_ref import valid_mask

OFFSET_LIMIT_32 = (1 << 31) - 2  # std::numeric_limits<int32_t>::max() - 1
TAKE_CAPACITY_MESSAGE = "Take operation overflowed binary array capacity"

DROP, EMIT_NULL = "drop", "emit_null"


def is_binary_like(t: pa.DataType) -> bool:
    return pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_binary(t) or pa.types.is_large_binary(t)


def offset_width(t: pa.DataType) -> int:
    return 8 if (pa.types.is_large_string(t) or pa.types.is_large_binary(t)) else 4


def byte_width(t: pa.DataType) -> int:
    """bytes per row of a fixed-width layout (the index type's for a dictionary)"""
    if pa.types.is_dictionary(t):
        return byte_width(t.index_type)
    if pa.types.is_fixed_size_binary(t):
        return t.byte_width
    return t.bit_width // 8


class Rows:
    """an array as rows: `data` is (n, W) uint8 for fixed width, a bool vector for bool, a list of bytes for binary"""

    def __init__(self, type, kind, data, valid, dictionary=None):
        self.type, self.kind, self.data, self.valid, self.dictionary = type, kind, data, np.asarray(valid, bool), dictionary

    def __len__(self):
        return len(self.valid)

    def pick(self, rows: np.ndarray, valid: np.ndarray) -> "Rows":
        """the rows at positions `rows` (an int64 vector) with validity `valid`"""
        if self.kind == "binary":
            data = [self.data[j] for j in rows.tolist()]
        else:
            data = self.data[rows]
        return Rows(self.type, self.kind, data, valid, self.dictionary)

    def null_count(self) -> int:
        return int((~self.valid).sum())


def from_arrow(arr: pa.Array) -> Rows:
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    t, n, off = arr.type, len(arr), arr.offset
    if pa.types.is_dictionary(t):
        r = from_arrow(arr.indices)
        return Rows(t, r.kind, r.data, r.valid, arr.dictionary)
    valid = valid_mask(arr)
    bufs = arr.buffers()
    if pa.types.is_boolean(t):
        if n == 0:
            return Rows(t, "bool", np.zeros(0, bool), valid)
        bits = np.unpackbits(np.frombuffer(bufs[1], np.uint8), bitorder="little")
        return Rows(t, "bool", bits[off:off + n].astype(bool), valid)
    if is_binary_like(t):
        if n == 0:
            return Rows(t, "binary", [], valid)
        o = np.frombuffer(bufs[1], np.int64 if offset_width(t) == 8 else np.int32, count=off + n + 1)[off:].astype(np.int64)
        chars = bufs[2].to_pybytes() if bufs[2] is not None else b""
        return Rows(t, "binary", [chars[o[i]:o[i + 1]] for i in range(n)], valid)
    w = byte_width(t)
    if n == 0:
        return Rows(t, "fixed", np.zeros((0, w), np.uint8), valid)
    data = np.frombuffer(bufs[1], np.uint8, count=(off + n) * w)[off * w:].reshape(n, w)
    return Rows(t, "fixed", data, valid)


def as_rows(x) -> Rows:
    return x if isinstance(x, Rows) else from_arrow(x)


# ---- the operations --------------------------------------------------------------------------------------------------
def selected(mask, null_selection=DROP) -> np.ndarray:
    """per mask row: is it kept"""
    m = as_rows(mask)
    assert m.kind == "bool", m.type
    if null_selection == DROP:
        return m.data & m.valid
    assert null_selection == EMIT_NULL, null_selection
    return m.data | ~m.valid


def filter_output_size(mask, null_selection=DROP) -> int:
    return int(selected(mask, null_selection).sum())


def filter(values, mask, null_selection=DROP) -> Rows:  # noqa: A001
    v, m = as_rows(values), as_rows(mask)
    if len(v) != len(m):
        raise pa.ArrowInvalid("Filter inputs must all be the same length")
    keep = np.flatnonzero(selected(m, null_selection))
    return v.pick(keep, v.valid[keep] & m.valid[keep])


def index_values(indices: Rows) -> list:
    """the indices as Python ints of their own signedness"""
    assert indices.kind == "fixed" and pa.types.is_integer(indices.type), indices.type
    dt = np.dtype(indices.type.to_pandas_dtype())
    return np.ascontiguousarray(indices.data).view(dt).reshape(-1).tolist()


def take(values, indices) -> Rows:
    v, ix = as_rows(values), as_rows(indices)
    idx = index_values(ix)
    n_values = len(v)
    for i, j in enumerate(idx):
        if ix.valid[i] and not 0 <= j < n_values:
            raise pa.ArrowIndexError(f"Index {j} out of bounds")
    rows = np.array([j if ok else 0 for j, ok in zip(idx, ix.valid.tolist())], np.int64)
    valid = ix.valid & (v.valid[rows] if n_values else np.zeros(len(ix), bool))
    if v.kind == "binary" and offset_width(v.type) == 4:
        sizes = [len(v.data[j]) for j, ok in zip(rows.tolist(), valid.tolist()) if ok]
        if take_overflows(sizes):
            raise pa.ArrowInvalid(TAKE_CAPACITY_MESSAGE)
    if n_values == 0:  # every index is null: nothing is read
        if v.kind == "binary":
            empty = [b""] * len(ix)
        elif v.kind == "bool":
            empty = np.zeros(len(ix), bool)
        else:
            empty = np.zeros((len(ix), byte_width(v.type)), np.uint8)
        return Rows(v.type, v.kind, empty, valid, v.dictionary)
    return v.pick(rows, valid)


def take_overflows(sizes) -> bool:
    """the int32-offset rule of the reference's VarBinary Take: fail once the running total of the taken (valid) rows'
    sizes exceeds 2^31 - 2.  Sizes are non-negative, so that is: the total exceeds 2^31 - 2."""
    total = 0
    for s in sizes:
        if total + s > OFFSET_LIMIT_32:
            return True
        total += s
    return False


def filter_overflows(sizes) -> bool:
    """Filter never fails on capacity (the reference's check is pruned from the filter path)"""
    return False


def take_indices(mask, null_selection=DROP) -> Rows:
    m = as_rows(mask)
    n = len(m)
    keep = np.flatnonzero(selected(m, null_selection))
    t, dt = (pa.uint16(), np.uint16) if n <= 0xFFFF else (pa.uint32(), np.uint32)
    data = keep.astype(dt).view(np.uint8).reshape(len(keep), dt().itemsize)
    return Rows(t, "fixed", data, m.valid[keep])


# ---- comparison ------------------------------------------------------------------------------------------------------
def row_mismatches(got: Rows, want: Rows) -> np.ndarray:
    """positions where validity differs, or both are valid and the row bytes differ"""
    assert len(got) == len(want), f"length {len(got)} != {len(want)}"
    bad = got.valid != want.valid
    both = got.valid & want.valid
    if want.kind == "binary":
        diff = np.array([g != w for g, w in zip(got.data, want.data)], bool) if len(want) else np.zeros(0, bool)
    elif want.kind == "bool":
        diff = got.data != want.data
    else:
        diff = (got.data != want.data).any(axis=1) if len(want) else np.zeros(0, bool)
    return np.flatnonzero(bad | (both & diff))


def _show(r: Rows, i: int) -> str:
    if not r.valid[i]:
        return "null"
    if r.kind == "fixed":
        return r.data[i].tobytes().hex()
    return repr(r.data[i])


def assert_rows_equal(got, want, msg=""):
    """validity equal, and the bytes equal at every valid slot (dictionaries: the same dictionary, indices byte for byte).
    `got` may be a pyarrow array (its type must equal want's) or Rows."""
    if isinstance(got, (pa.Array, pa.ChunkedArray)):
        assert got.type == want.type, f"{msg}: type {got.type} != {want.type}"
    g = as_rows(got)
    assert g.kind == want.kind, f"{msg}: {g.kind} != {want.kind}"
    if want.dictionary is not None:
        assert g.dictionary is not None and g.dictionary.equals(want.dictionary), f"{msg}: dictionary differs"
    assert len(g) == len(want), f"{msg}: length {len(g)} != {len(want)}"
    bad = row_mismatches(g, want)
    if len(bad):
        show = bad[:5].tolist()
        raise AssertionError(f"{msg}: {len(bad)} of {len(want)} rows differ, at {show}: got {[_show(g, i) for i in show]} "
                             f"want {[_show(want, i) for i in show]}")
