"""CPU oracle: a numpy restatement of the reference's algorithms for the hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under arrow_b200/ imports this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may.

Parity status: PINNED.  tests/test_oracle.py checks every function here against
  (a) the reference's own known-answer vectors transcribed in tests/golden/kat.json
      (vector_selection_test.cc, vector_sort_test.cc, scalar_cast_test.cc,
       scalar_arithmetic_test.cc, grouper_test.cc, hash_aggregate_test.cc), and
  (b) the reference binary itself (pyarrow 24.0.0 = libarrow_compute.so.2400, the same
      kernels as /root/reference for this path, SURVEY.md section 8c) on seeded random inputs.

pyarrow is used as the host array container only (buffers in, buffers out); every
computation below is plain numpy over Arrow's buffer layout.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

# ---------------------------------------------------------------------------------------
# buffer-level helpers (Arrow columnar format: LSB-first bitmaps, offset in elements)
# ---------------------------------------------------------------------------------------
_NP = {pa.int8(): np.int8, pa.uint8(): np.uint8, pa.int16(): np.int16, pa.uint16(): np.uint16,
       pa.int32(): np.int32, pa.uint32(): np.uint32, pa.int64(): np.int64, pa.uint64(): np.uint64,
       pa.float32(): np.float32, pa.float64(): np.float64}


def np_dtype(t: pa.DataType):
    if t in _NP:
        return _NP[t]
    if pa.types.is_date32(t) or pa.types.is_time32(t):
        return np.int32
    if pa.types.is_date64(t) or pa.types.is_time64(t) or pa.types.is_timestamp(t) or pa.types.is_duration(t):
        return np.int64
    raise NotImplementedError(str(t))


def bits(buf, offset: int, length: int) -> np.ndarray:
    """bool[length] view of an LSB-first bitmap (util/bit_util.h GetBit)."""
    if buf is None:
        return np.ones(length, dtype=bool)
    raw = np.frombuffer(buf, dtype=np.uint8)
    return np.unpackbits(raw, bitorder="little")[offset:offset + length].astype(bool)


def validity(arr: pa.Array) -> np.ndarray:
    if arr.null_count == 0:
        return np.ones(len(arr), dtype=bool)
    return bits(arr.buffers()[0], arr.offset, len(arr))


def values(arr: pa.Array) -> np.ndarray:
    """Fixed-width data buffer as numpy (slots under nulls included), or bool for boolean."""
    if pa.types.is_dictionary(arr.type):
        return values(arr.indices)
    if pa.types.is_boolean(arr.type):
        return bits(arr.buffers()[1], arr.offset, len(arr))
    dt = np_dtype(arr.type)
    buf = arr.buffers()[1]
    if buf is None or len(arr) == 0:
        return np.zeros(0, dtype=dt)
    return np.frombuffer(buf, dtype=dt)[arr.offset:arr.offset + len(arr)]


def make_array(t: pa.DataType, vals: np.ndarray, valid: np.ndarray | None = None) -> pa.Array:
    if pa.types.is_boolean(t):
        return pa.array(vals.astype(bool), type=t, mask=None if valid is None else ~valid)
    dt = np_dtype(t)
    vals = np.ascontiguousarray(vals, dtype=dt)
    if valid is None or valid.all():
        vbuf, nc = None, 0
    else:
        vbuf = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
        nc = int((~valid).sum())
    return pa.Array.from_buffers(t, len(vals), [vbuf, pa.py_buffer(vals.tobytes())], null_count=nc)


def strings(arr: pa.Array):
    """(offsets int64[n+1] rebased to the slice, bytes uint8[]) of a (large_)utf8/binary array."""
    ow = np.int64 if (pa.types.is_large_string(arr.type) or pa.types.is_large_binary(arr.type)) else np.int32
    offs = np.frombuffer(arr.buffers()[1], dtype=ow)[arr.offset:arr.offset + len(arr) + 1].astype(np.int64)
    data = np.frombuffer(arr.buffers()[2], dtype=np.uint8) if arr.buffers()[2] is not None else np.zeros(0, np.uint8)
    return offs, data


def make_strings(t: pa.DataType, lengths: np.ndarray, data: np.ndarray, valid: np.ndarray | None) -> pa.Array:
    ow = np.int64 if (pa.types.is_large_string(t) or pa.types.is_large_binary(t)) else np.int32
    offs = np.zeros(len(lengths) + 1, dtype=np.int64)
    np.cumsum(lengths, out=offs[1:])
    if ow == np.int32 and offs[-1] > 2**31 - 2:
        raise pa.ArrowInvalid("Take operation overflowed binary array capacity")
    if valid is None or valid.all():
        vbuf, nc = None, 0
    else:
        vbuf = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
        nc = int((~valid).sum())
    return pa.Array.from_buffers(t, len(lengths), [vbuf, pa.py_buffer(offs.astype(ow).tobytes()),
                                                   pa.py_buffer(np.ascontiguousarray(data).tobytes())], null_count=nc)


def _gather_strings(arr: pa.Array, idx: np.ndarray, out_valid: np.ndarray) -> pa.Array:
    offs, data = strings(arr)
    starts = offs[:-1][idx]
    lens = (offs[1:] - offs[:-1])[idx]
    lens = np.where(out_valid, lens, 0)
    total = int(lens.sum())
    out_offs = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum(lens, out=out_offs[1:])
    # byte gather: position p of the output belongs to string k = searchsorted
    if total:
        k = np.repeat(np.arange(len(idx)), lens)
        within = np.arange(total) - out_offs[:-1][k]
        out = data[starts[k] + within]
    else:
        out = np.zeros(0, np.uint8)
    return make_strings(arr.type, lens, out, out_valid)


def _is_binary(t):
    return pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t) or pa.types.is_large_binary(t)


# ---------------------------------------------------------------------------------------
# Filter   (kernels/vector_selection_filter_internal.cc:62-114, 158-510, 552-856)
# ---------------------------------------------------------------------------------------
def filter_selection(mask: pa.Array, null_selection: str):
    """(selected rows bool[n], emitted-as-null bool[n]) -- GetFilterOutputSize's two cases."""
    d, v = values(mask), validity(mask)
    if null_selection == "drop":
        return d & v, np.zeros(len(mask), dtype=bool)
    return d | ~v, ~v


def filter(vals: pa.Array, mask: pa.Array, null_selection: str = "drop") -> pa.Array:
    if len(vals) != len(mask):
        raise pa.ArrowInvalid("Filter inputs must all be the same length")
    sel, emit = filter_selection(mask, null_selection)
    idx = np.nonzero(sel)[0]
    out_valid = validity(vals)[idx] & ~emit[idx]
    if pa.types.is_dictionary(vals.type):
        ind = make_array(vals.type.index_type, values(vals)[idx], out_valid)
        return pa.DictionaryArray.from_arrays(ind, vals.dictionary)
    if _is_binary(vals.type):
        return _gather_strings(vals, idx, out_valid)
    return make_array(vals.type, values(vals)[idx], out_valid)


def take_indices_from_filter(mask: pa.Array, null_selection: str = "drop") -> pa.Array:
    """GetTakeIndices (kernels/vector_selection_take_internal.cc:62-305)."""
    sel, emit = filter_selection(mask, null_selection)
    idx = np.nonzero(sel)[0]
    t = pa.uint16() if len(mask) <= 0xFFFF else pa.uint32()
    return make_array(t, idx, ~emit[idx])


# ---------------------------------------------------------------------------------------
# Take   (kernels/vector_selection_take_internal.cc:336-497, gather_internal.h:84-251)
# ---------------------------------------------------------------------------------------
def take(vals: pa.Array, indices: pa.Array, boundscheck: bool = True) -> pa.Array:
    iv = validity(indices)
    idx = values(indices).astype(np.int64) if indices.type != pa.uint64() else values(indices)
    n = len(vals)
    bad = iv & ((idx < 0) | (idx >= n)) if idx.dtype != np.uint64 else iv & (idx >= np.uint64(n))
    if bad.any():
        # CheckIndexBounds, util/int_util.cc:554-555
        raise pa.ArrowIndexError(f"Index {int(values(indices)[np.nonzero(bad)[0][0]])} out of bounds")
    safe = np.where(iv, idx, 0).astype(np.int64)
    if n == 0:
        safe = np.zeros(len(indices), dtype=np.int64)
        out_valid = np.zeros(len(indices), dtype=bool)
        gathered_valid = out_valid
    else:
        gathered_valid = validity(vals)[safe]
        out_valid = iv & gathered_valid
    if pa.types.is_dictionary(vals.type):
        data = values(vals)[safe] if n else np.zeros(len(indices), np_dtype(vals.type.index_type))
        ind = make_array(vals.type.index_type, np.where(out_valid, data, 0), out_valid)
        return pa.DictionaryArray.from_arrays(ind, vals.dictionary)
    if _is_binary(vals.type):
        return _gather_strings(vals, safe, out_valid)
    if pa.types.is_boolean(vals.type):
        return make_array(vals.type, values(vals)[safe] & out_valid, out_valid)
    data = values(vals)[safe] if n else np.zeros(len(indices), np_dtype(vals.type))
    return make_array(vals.type, np.where(iv, data, 0), out_valid)


# ---------------------------------------------------------------------------------------
# Cast   (kernels/scalar_cast_numeric.cc:45-279, scalar_cast_internal.cc:41-53)
# ---------------------------------------------------------------------------------------
def cast(arr: pa.Array, to: pa.DataType, safe: bool = True) -> pa.Array:
    v, valid = values(arr), validity(arr)
    src, dst = np_dtype(arr.type), np_dtype(to)
    si, di = np.issubdtype(src, np.integer), np.issubdtype(dst, np.integer)
    with np.errstate(all="ignore"):
        if not si and di:
            # static_cast of out-of-range floats is UB in C++; only in-range values are pinned
            fin = np.isfinite(v)
            lim_lo, lim_hi = float(np.iinfo(dst).min), float(np.iinfo(dst).max)
            inr = fin & (np.trunc(v) >= lim_lo) & (np.trunc(v) <= lim_hi)
            # float(int64 max) rounds up to 2^63: exclude it explicitly
            if dst in (np.int64, np.uint64):
                inr &= np.trunc(v) < float(2**63 if dst == np.int64 else 2**64)
            out = np.zeros(len(v), dtype=dst)
            out[inr] = np.trunc(v[inr]).astype(dst)
            if safe:
                bad = valid & (~inr | (out.astype(src) != v))
                if bad.any():
                    x = v[np.nonzero(bad)[0][0]]
                    text = ("-nan" if np.signbit(x) else "nan") if np.isnan(x) else f"{x:f}"  # printf's %f
                    raise pa.ArrowInvalid(f"Float value {text} was truncated converting to {to}")
            return make_array(to, out, valid), (inr | ~valid)
        out = v.astype(dst)
    if safe and si and di:
        lo = max(int(np.iinfo(src).min), int(np.iinfo(dst).min))
        hi = min(int(np.iinfo(src).max), int(np.iinfo(dst).max))
        vi = v.astype(object) if src == np.uint64 else v
        bad = valid & np.array([(int(x) < lo or int(x) > hi) for x in vi], dtype=bool) if src == np.uint64 else \
            valid & ((v < lo) | (v > hi))
        if bad.any():
            raise pa.ArrowInvalid(f"Integer value {int(v[np.nonzero(bad)[0][0]])} not in range: {lo} to {hi}")
    if safe and si and not di and src().itemsize >= 4 and not (src().itemsize == 4 and dst == np.float64):
        limit = 1 << 24 if dst == np.float32 else 1 << 53
        lo = -limit if np.issubdtype(src, np.signedinteger) else 0
        lo = max(lo, int(np.iinfo(src).min))
        hi = min(limit, int(np.iinfo(src).max))
        bad = valid & ((v < lo) | (v > hi)) if src != np.uint64 else valid & (v > np.uint64(hi))
        if bad.any():
            raise pa.ArrowInvalid(f"Integer value {int(v[np.nonzero(bad)[0][0]])} not in range: {lo} to {hi}")
    return make_array(to, out, valid), np.ones(len(v), dtype=bool)


def cast_array(arr, to, safe=True) -> pa.Array:
    return cast(arr, to, safe)[0]


# ---------------------------------------------------------------------------------------
# Arithmetic / compare   (kernels/base_arithmetic_internal.h:44-423, codegen_internal.h:813-976,
#                         codegen_internal.cc:166-218 CommonNumeric, scalar_compare.cc:42-303)
# ---------------------------------------------------------------------------------------
def common_numeric(types):
    if any(t == pa.float64() for t in types):
        return pa.float64()
    if any(t == pa.float32() for t in types):
        return pa.float32()
    ms = max([t.bit_width for t in types if pa.types.is_signed_integer(t)], default=0)
    mu = max([t.bit_width for t in types if pa.types.is_unsigned_integer(t)], default=0)
    if ms == 0:
        return {8: pa.uint8(), 16: pa.uint16(), 32: pa.uint32()}.get(mu, pa.uint64())
    if ms <= mu:
        ms = 1 << (mu).bit_length()
    return {8: pa.int8(), 16: pa.int16(), 32: pa.int32()}.get(ms, pa.int64())


def _operand(x, t, n):
    """-> (values ndarray[n], valid ndarray[n]) of an array or a broadcast scalar, cast to t."""
    if isinstance(x, pa.Array):
        if x.type != t:
            x = cast_array(x, t, safe=True)
        return values(x), validity(x)
    s = x if isinstance(x, pa.Scalar) else pa.scalar(x)
    dt = np_dtype(t)
    if not s.is_valid:
        return np.zeros(n, dtype=dt), np.zeros(n, dtype=bool)
    # the scalar goes through the same safe cast as an array operand (its exact bits when the type already matches)
    one = values(cast_array(pa.array([s], s.type), t, safe=True) if s.type != t else pa.array([s], s.type))
    return np.repeat(one, n), np.ones(n, dtype=bool)


def _binary_prepare(l, r):
    types = [x.type if isinstance(x, (pa.Array, pa.Scalar)) else pa.scalar(x).type for x in (l, r)]
    t = types[0] if types[0] == types[1] else common_numeric(types)
    n = len(l) if isinstance(l, pa.Array) else len(r)
    if isinstance(l, pa.Array) and isinstance(r, pa.Array) and len(l) != len(r):
        raise pa.ArrowInvalid("Array arguments must all be the same length")
    (a, va), (b, vb) = _operand(l, t, n), _operand(r, t, n)
    return t, a, b, va & vb


def arithmetic(op: str, l, r) -> pa.Array:
    t, a, b, valid = _binary_prepare(l, r)
    dt = np_dtype(t)
    checked = op.endswith("_checked")
    base = op.replace("_checked", "")
    with np.errstate(all="ignore"):
        if np.issubdtype(dt, np.floating):
            if base == "add":
                out = a + b
            elif base == "subtract":
                out = a - b
            elif base == "multiply":
                out = a * b
            else:
                if checked and (valid & (b == 0)).any():
                    raise pa.ArrowInvalid("divide by zero")
                out = a / b
            return make_array(t, out, valid)
        info = np.iinfo(dt)
        A, B = a.astype(object), b.astype(object)  # exact python ints
        if base == "add":
            exact = A + B
        elif base == "subtract":
            exact = A - B
        elif base == "multiply":
            exact = A * B
        else:
            bb = np.where(b == 0, 1, b).astype(object)
            # C++ division truncates toward zero
            exact = np.array([int(abs(x) // abs(y)) * (1 if (x >= 0) == (y >= 0) else -1) for x, y in zip(A, bb)],
                             dtype=object)
            ovf = np.array([not (info.min <= int(e) <= info.max) for e in exact], dtype=bool) & (b != 0)
            # every row runs and each failing one overwrites the status (ScalarBinaryNotNullStateful): the LAST
            # offending valid row decides between the two messages
            bad = np.flatnonzero(valid & ((b == 0) | (ovf if checked else False)))
            if len(bad):
                raise pa.ArrowInvalid("divide by zero" if b[bad[-1]] == 0 else "overflow")
            exact = np.where(ovf, 0, exact)  # Divide: INT_MIN / -1 -> 0
            exact = np.where(b == 0, 0, exact)
        if len(exact):
            ovf = np.array([not (info.min <= int(e) <= info.max) for e in exact], dtype=bool)
            if checked and (valid & ovf).any():
                raise pa.ArrowInvalid("overflow")
            span = 1 << (8 * dt().itemsize)
            wrapped = np.array([((int(e) - info.min) % span) + info.min for e in exact], dtype=object)
            out = wrapped.astype(dt)
        else:
            out = np.zeros(0, dtype=dt)
    return make_array(t, out, valid)


def compare(op: str, l, r) -> pa.Array:
    t, a, b, valid = _binary_prepare(l, r)
    with np.errstate(all="ignore"):
        out = {"equal": a == b, "not_equal": a != b, "greater": a > b, "greater_equal": a >= b,
               "less": a < b, "less_equal": a <= b}[op]
    return make_array(pa.bool_(), out, valid)


# ---------------------------------------------------------------------------------------
# boolean logic + validity predicates
#   (kernels/scalar_boolean.cc:30-270 AndOp/OrOp/XorOp/AndNotOp/InvertOp + Kleene*Op,
#    kernels/scalar_validity.cc:35-311 IsValidExec/IsNullExec/TrueUnlessNullExec/is_nan)
# ---------------------------------------------------------------------------------------
def _bool_operand(x, n):
    if isinstance(x, pa.Array):
        return values(x), validity(x)
    s = x if isinstance(x, pa.Scalar) else pa.scalar(x, pa.bool_())
    if not s.is_valid:
        return np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    return np.full(n, bool(s.as_py())), np.ones(n, dtype=bool)


def boolean(op: str, l, r=None) -> pa.Array:
    n = len(l) if isinstance(l, pa.Array) else len(r)
    a, va = _bool_operand(l, n)
    if op == "invert":
        return make_array(pa.bool_(), ~a, va)
    b, vb = _bool_operand(r, n)
    if op == "and":
        return make_array(pa.bool_(), a & b, va & vb)
    if op == "or":
        return make_array(pa.bool_(), a | b, va & vb)
    if op == "xor":
        return make_array(pa.bool_(), a ^ b, va & vb)
    if op == "and_not":
        return make_array(pa.bool_(), a & ~b, va & vb)
    if op == "and_kleene":      # false AND anything = false (scalar_boolean.cc:138-210)
        return make_array(pa.bool_(), a & b, (va & vb) | (va & ~a) | (vb & ~b))
    if op == "or_kleene":       # true OR anything = true
        return make_array(pa.bool_(), a | b, (va & vb) | (va & a) | (vb & b))
    if op == "and_not_kleene":
        return make_array(pa.bool_(), a & ~b, (va & vb) | (va & ~a) | (vb & b))
    raise NotImplementedError(op)


def validity_op(op: str, arr: pa.Array, nan_is_null: bool = False) -> pa.Array:
    valid = validity(arr)
    if op == "is_valid":
        return make_array(pa.bool_(), valid)
    if op == "true_unless_null":
        return make_array(pa.bool_(), np.ones(len(arr), dtype=bool), valid)
    nan = np.zeros(len(arr), dtype=bool)
    if pa.types.is_floating(arr.type):
        with np.errstate(all="ignore"):
            nan = np.isnan(values(arr))
    if op == "is_null":
        return make_array(pa.bool_(), ~valid | (nan & valid if nan_is_null else False))
    if op == "is_nan":
        return make_array(pa.bool_(), nan, valid)
    raise NotImplementedError(op)


def if_else(cond, left, right) -> pa.Array:
    """if_else (kernels/scalar_if_else.cc:62-520): out = cond ? left : right; valid = cond valid AND the chosen side's
    validity.  Numeric left / right are promoted to CommonNumeric first (scalar_if_else.cc:1227-1266)."""
    n = next(len(x) for x in (cond, left, right) if isinstance(x, pa.Array))
    c, vc = _bool_operand(cond, n)
    sides = [x if isinstance(x, (pa.Array, pa.Scalar)) else pa.scalar(x) for x in (left, right)]
    if all(pa.types.is_boolean(x.type) for x in sides):
        (l, vl), (r, vr) = (_bool_operand(x, n) for x in sides)
        return make_array(pa.bool_(), np.where(c, l, r), vc & np.where(c, vl, vr))
    t = sides[0].type if sides[0].type == sides[1].type else common_numeric([x.type for x in sides])
    cols = [_operand(x, t, n) for x in sides]   # the implicit safe cast of arithmetic / compare
    (l, vl), (r, vr) = cols
    return make_array(t, np.where(c, l, r), vc & np.where(c, vl, vr))


# ---------------------------------------------------------------------------------------
# SortIndices   (kernels/vector_array_sort.cc:144-178,524-540; vector_sort_internal.h:113-305)
# ---------------------------------------------------------------------------------------
def sort_indices(arr: pa.Array, order: str = "ascending", null_placement: str = "at_end") -> pa.Array:
    v, valid = values(arr), validity(arr)
    idx = np.arange(len(arr), dtype=np.uint64)
    is_nan = np.zeros(len(arr), dtype=bool)
    if np.issubdtype(v.dtype, np.floating):
        is_nan = valid & np.isnan(v)
    nulls = idx[~valid]               # stable partition keeps index order
    nans = idx[is_nan]
    rest = idx[valid & ~is_nan]
    keys = v[valid & ~is_nan]
    if np.issubdtype(keys.dtype, np.floating):
        keys = keys + 0.0             # -0.0 == +0.0 under operator<
    if order == "ascending":
        perm = np.argsort(keys, kind="stable")
    else:
        # stable descending: comparator is `rhs < lhs`; equal keys keep index order
        if np.issubdtype(keys.dtype, np.floating):
            perm = np.argsort(-keys, kind="stable")
        elif np.issubdtype(keys.dtype, np.signedinteger):
            perm = np.argsort(~keys, kind="stable")      # ~x = -x-1 reverses order without overflow
        else:
            perm = np.argsort(np.iinfo(keys.dtype).max - keys, kind="stable")
    rest = rest[perm]
    out = np.concatenate([rest, nans, nulls] if null_placement == "at_end" else [nulls, nans, rest])
    return make_array(pa.uint64(), out)


def select_k_unstable(arr: pa.Array, k: int, order: str = "ascending", null_placement: str = "at_end") -> pa.Array:
    """select_k_unstable (ArraySelector, kernels/vector_select_k.cc:157-232): the first k rows of the sort order.  The
    reference's selection is unstable (ties in any order); this restatement -- like the CUDA path -- returns the stable
    sort's prefix, one of the permitted answers.  NaNs / nulls follow the values as in sort_indices (the installed
    24.0.0 binary never selects them; /root/reference does, per null_placement)."""
    if k < 0:
        raise pa.ArrowInvalid(f"select_k_unstable requires a nonnegative `k`, got {k}")
    return sort_indices(arr, order, null_placement).slice(0, min(k, len(arr)))


def sort_indices_multi(columns, sort_keys, null_placement: str = "at_end") -> pa.Array:
    """SortIndices over a record batch (kernels/vector_sort.cc:386-600): lexicographic over sort_keys = [(name, order)],
    stable.  Restated as the reference's own fallback states it -- a stable sort per key from the least significant key
    to the most significant one, each with the single-key rules of sort_indices above (nulls, then NaNs, compare equal
    among themselves)."""
    n = len(next(iter(columns.values())))
    perm = np.arange(n, dtype=np.uint64)
    for name, order in reversed(list(sort_keys)):
        col = columns[name].take(pa.array(perm))
        perm = perm[values(sort_indices(col, order, null_placement)).astype(np.int64)]
    return pa.array(perm, pa.uint64())


# ---------------------------------------------------------------------------------------
# Grouper   (compute/row/grouper.cc:555-963; semantics per grouper_test.cc:678-760)
# ---------------------------------------------------------------------------------------
class Grouper:
    """ids in first-occurrence order; a null key is its own group; keys compare by bytes."""

    def __init__(self, key_types):
        self.key_types = list(key_types)
        self.table = {}
        self.uniques = []  # list of tuples (per column: bytes or None)

    def _rows(self, keys):
        # one bytes object per key value: the raw little-endian bytes of a fixed-width value, the bytes of a
        # utf8 / binary value (row/encode_internal.cc encodes both into the row; var-length ones with their length)
        cols = []
        for k in keys:
            valid = validity(k)
            if _is_binary(k.type):
                offs, data = strings(k)
                raw = [data[offs[i]:offs[i + 1]].tobytes() for i in range(len(k))]
            else:
                v = values(k)
                raw = v.view(np.uint8).reshape(len(v), -1) if len(v) else np.zeros((0, 1), np.uint8)
                raw = [raw[i].tobytes() for i in range(len(v))]
            cols.append((raw, valid))
        for i in range(len(keys[0])):
            yield tuple(raw[i] if valid[i] else None for raw, valid in cols)

    def consume(self, keys) -> pa.Array:
        if isinstance(keys, pa.Array):
            keys = [keys]
        ids = np.zeros(len(keys[0]), dtype=np.uint32)
        for i, row in enumerate(self._rows(keys)):
            g = self.table.get(row)
            if g is None:
                g = self.table[row] = len(self.uniques)
                self.uniques.append(row)
            ids[i] = g
        return make_array(pa.uint32(), ids)

    def lookup(self, keys) -> pa.Array:
        if isinstance(keys, pa.Array):
            keys = [keys]
        ids = np.zeros(len(keys[0]), dtype=np.uint32)
        ok = np.zeros(len(keys[0]), dtype=bool)
        for i, row in enumerate(self._rows(keys)):
            g = self.table.get(row)
            if g is not None:
                ids[i], ok[i] = g, True
        return make_array(pa.uint32(), ids, ok)

    @property
    def num_groups(self):
        return len(self.uniques)

    def get_uniques(self):
        out = []
        for j, t in enumerate(self.key_types):
            valid = np.array([u[j] is not None for u in self.uniques], dtype=bool)
            if _is_binary(t):
                lens = np.array([len(u[j]) if u[j] is not None else 0 for u in self.uniques], dtype=np.int64)
                data = np.frombuffer(b"".join(u[j] for u in self.uniques if u[j] is not None), dtype=np.uint8)
                out.append(make_strings(t, lens, data, valid))
                continue
            dt = np_dtype(t)
            vals = np.array([np.frombuffer(u[j], dtype=dt)[0] if u[j] is not None else 0 for u in self.uniques],
                            dtype=dt)
            out.append(make_array(t, vals, valid))
        return out


# ---------------------------------------------------------------------------------------
# Ungrouped aggregates   (kernels/aggregate_basic.inc.cc:49-107 SumImpl, :227-290 MeanImpl,
# :657-701 MinMaxState, :776-860 MinMaxImpl; kernels/aggregate_basic.cc:98-130 CountImpl)
# ---------------------------------------------------------------------------------------
def _agg_acc(t):
    if pa.types.is_floating(t):
        return pa.float64(), np.float64
    return (pa.int64(), np.int64) if pa.types.is_signed_integer(t) else (pa.uint64(), np.uint64)


def scalar_sum(arr: pa.Array, skip_nulls=True, min_count=1) -> pa.Scalar:
    v, valid = values(arr), validity(arr)
    out_t, acc = _agg_acc(arr.type)
    n_valid = int(valid.sum())
    if (not skip_nulls and n_valid < len(arr)) or n_valid < min_count:
        return pa.scalar(None, out_t)
    with np.errstate(over="ignore"):
        total = v[valid].astype(acc).sum(dtype=acc)  # integers wrap; floats: numpy's pairwise sum
    return pa.scalar(total.item(), out_t)


def scalar_mean(arr: pa.Array, skip_nulls=True, min_count=1) -> pa.Scalar:
    valid = validity(arr)
    n_valid = int(valid.sum())
    if (not skip_nulls and n_valid < len(arr)) or n_valid < min_count:
        return pa.scalar(None, pa.float64())
    with np.errstate(invalid="ignore", divide="ignore"):  # 0 valid values and min_count == 0 -> 0/0 = NaN (:272-283)
        return pa.scalar(float(values(arr)[valid].astype(np.float64).sum() / np.float64(n_valid)), pa.float64())  # double accumulator (:263-268)


def scalar_min_max(arr: pa.Array, skip_nulls=True, min_count=1) -> pa.Scalar:
    v, valid = values(arr), validity(arr)
    st = pa.struct([("min", arr.type), ("max", arr.type)])
    n_valid = int(valid.sum())
    if (n_valid < len(arr) and not skip_nulls) or n_valid < max(1, min_count):
        return pa.scalar({"min": None, "max": None}, st)
    vv = v[valid]
    if pa.types.is_floating(arr.type):  # std::fmin / std::fmax starting from NaN: NaNs are ignored
        lo, hi = (np.nan, np.nan) if np.isnan(vv).all() else (np.nanmin(vv), np.nanmax(vv))
    else:
        lo, hi = vv.min(), vv.max()
    return pa.scalar({"min": lo.item() if hasattr(lo, "item") else lo, "max": hi.item() if hasattr(hi, "item") else hi}, st)


def scalar_count(arr: pa.Array, mode="only_valid") -> pa.Scalar:
    n_valid = int(validity(arr).sum())
    return pa.scalar({"only_valid": n_valid, "only_null": len(arr) - n_valid, "all": len(arr)}[mode], pa.int64())


# ---------------------------------------------------------------------------------------
# unique / value_counts / dictionary_encode   (kernels/vector_hash.cc:65-235, 782-830)
# The memo table hands out indices in first-occurrence order (RegularHashKernel::DoAppend,
# vector_hash.cc:300-340); UniqueAction and ValueCountsAction encode null as a value,
# DictEncodeAction only with DictionaryEncodeOptions::ENCODE (api_vector.h:66-82).
# ---------------------------------------------------------------------------------------
def _memo(arr: pa.Array, encode_nulls: bool):
    if _is_binary(arr.type):  # BinaryMemoTable: the same first-occurrence indices over the value bytes
        valid = validity(arr)
        offs, data = strings(arr)
        table, order, idx = {}, [], np.zeros(len(arr), dtype=np.int32)
        for i in range(len(arr)):
            if not valid[i] and not encode_nulls:
                continue
            key = data[offs[i]:offs[i + 1]].tobytes() if valid[i] else None
            g = table.get(key)
            if g is None:
                g = table[key] = len(order)
                order.append(i)
            idx[i] = g
        order = np.array(order, dtype=np.int64)
        uniq_valid = valid[order] if len(order) else np.zeros(0, bool)
        return idx, _gather_strings(arr, order, uniq_valid)
    v, valid = values(arr), validity(arr)
    raw = v.view(np.uint8).reshape(len(v), -1) if len(v) else np.zeros((0, 1), np.uint8)
    table, order, idx = {}, [], np.zeros(len(v), dtype=np.int32)
    for i in range(len(v)):
        if not valid[i] and not encode_nulls:
            continue
        key = raw[i].tobytes() if valid[i] else None
        g = table.get(key)
        if g is None:
            g = table[key] = len(order)
            order.append(i)
        idx[i] = g
    order = np.array(order, dtype=np.int64)
    uniq_valid = valid[order] if len(order) else np.zeros(0, bool)
    uniq = make_array(arr.type, v[order] if len(order) else v[:0], uniq_valid)
    return idx, uniq


def unique(arr: pa.Array) -> pa.Array:
    return _memo(arr, True)[1]


def value_counts(arr: pa.Array) -> pa.StructArray:
    idx, uniq = _memo(arr, True)
    counts = np.bincount(idx, minlength=len(uniq)).astype(np.int64)
    return pa.StructArray.from_arrays([uniq, make_array(pa.int64(), counts)], names=["values", "counts"])


def dictionary_encode(arr: pa.Array, null_encoding: str = "mask") -> pa.DictionaryArray:
    encode = null_encoding == "encode"
    idx, uniq = _memo(arr, encode)
    idx_valid = None if encode else validity(arr)
    return pa.DictionaryArray.from_arrays(make_array(pa.int32(), idx, idx_valid), uniq)


# ---------------------------------------------------------------------------------------
# Hash aggregates   (kernels/hash_aggregate_numeric.cc:44-434, kernels/hash_aggregate.cc:61-420)
# ---------------------------------------------------------------------------------------
def _sum_type(t):
    if pa.types.is_signed_integer(t):
        return pa.int64()
    if pa.types.is_unsigned_integer(t):
        return pa.uint64()
    return pa.float64()


def hash_aggregate(function: str, vals, ids: pa.Array, num_groups: int, *, skip_nulls=True, min_count=1,
                   mode="only_valid") -> pa.Array:
    g = values(ids).astype(np.int64)
    if function == "hash_count_all":
        return make_array(pa.int64(), np.bincount(g, minlength=num_groups).astype(np.int64))
    if function == "hash_count_distinct":
        # GroupedCountDistinctImpl (hash_aggregate.cc:1400-1478): a Grouper over (value, group id); Finalize counts the
        # distinct pairs per group that CountOptions::mode admits (a null is one more distinct value under "all")
        pairs = Grouper([vals.type, pa.uint32()])
        pairs.consume([vals, ids])
        uv, ug = pairs.get_uniques()
        ok, gg = validity(uv), values(ug).astype(np.int64)
        sel = ok if mode == "only_valid" else (~ok if mode == "only_null" else np.ones(len(gg), bool))
        return make_array(pa.int64(), np.bincount(gg[sel], minlength=num_groups).astype(np.int64))
    v, valid = values(vals), validity(vals)
    if function == "hash_count":
        sel = valid if mode == "only_valid" else (~valid if mode == "only_null" else np.ones(len(g), bool))
        return make_array(pa.int64(), np.bincount(g[sel], minlength=num_groups).astype(np.int64))
    counts = np.bincount(g[valid], minlength=num_groups).astype(np.int64)
    saw_null = np.bincount(g[~valid], minlength=num_groups) > 0
    ok = counts >= min_count
    if not skip_nulls:
        ok &= ~saw_null
    if function == "hash_sum":
        t = _sum_type(vals.type)
        dt = np_dtype(t)
        acc = np.zeros(num_groups, dtype=dt)
        with np.errstate(all="ignore"):
            np.add.at(acc, g[valid], v[valid].astype(dt))  # row order; integer adds wrap
        return make_array(t, acc, ok)
    if function == "hash_product":   # GroupedProductImpl, hash_aggregate_numeric.cc:311-335: integers wrap mod 2^64
        t = _sum_type(vals.type)
        dt = np_dtype(t)
        acc = np.ones(num_groups, dtype=dt)
        with np.errstate(all="ignore"):
            np.multiply.at(acc, g[valid], v[valid].astype(dt))
        return make_array(t, acc, ok)
    if function in ("hash_any", "hash_all"):   # GroupedBooleanAggregator, hash_aggregate.cc:1232-1397
        hit = v[valid] if function == "hash_any" else ~v[valid]
        seen = np.bincount(g[valid][hit], minlength=num_groups) > 0
        out = seen if function == "hash_any" else ~seen
        ok = counts >= min_count
        if not skip_nulls:   # a null leaves the group undecided unless the value is already forced (Kleene)
            ok &= ~saw_null | (out if function == "hash_any" else ~out)
        return make_array(pa.bool_(), out, ok)
    if function == "hash_mean":
        acc = np.zeros(num_groups, dtype=np.float64)
        np.add.at(acc, g[valid], v[valid].astype(np.float64))
        with np.errstate(all="ignore"):  # a group without values and min_count == 0 is 0/0 = NaN (:402-421)
            mean = np.where(ok, acc / counts, 0.0)
        return make_array(pa.float64(), mean, ok)
    if function in ("hash_min", "hash_max"):
        # AntiExtrema<T> (hash_aggregate.cc:305-309): integers start at the type's max / min, floats at NaN, which
        # std::fmin / fmax replace with the first non-NaN value -- a group whose values are all NaN stays NaN.  NaNs are
        # dropped here before reducing: np.fmin.at's vectorised loops do not skip a signalling NaN on every host CPU
        dt = v.dtype
        flt = np.issubdtype(dt, np.floating)
        sel = valid & ~np.isnan(v) if flt else valid
        info = np.finfo(dt) if flt else np.iinfo(dt)
        acc = np.full(num_groups, (np.inf if flt else info.max) if function == "hash_min" else (-np.inf if flt else info.min), dt)
        (np.minimum if function == "hash_min" else np.maximum).at(acc, g[sel], v[sel])
        if flt:
            acc[np.bincount(g[sel], minlength=num_groups) == 0] = np.nan
        ok = counts > 0
        if not skip_nulls:
            ok &= ~saw_null
        return make_array(vals.type, acc, ok)
    raise NotImplementedError(function)


def group_by(keys, aggregates):
    """acero aggregate node over one batch (groupby_aggregate_node.cc:210-337)."""
    if isinstance(keys, pa.Array):
        keys = [keys]
    gr = Grouper([k.type for k in keys])
    ids = gr.consume(keys)
    outs = [hash_aggregate(fn, vals, ids, gr.num_groups, **(opts or {})) for fn, vals, opts in aggregates]
    return gr.get_uniques(), outs


# ---------------------------------------------------------------------------------------
# Hash join: the matching row pairs   (acero/hash_join_node.cc, acero/swiss_join.cc; JoinType acero/options.h:365-374;
# JoinKeyCmp::EQ: a null key matches nothing)
# ---------------------------------------------------------------------------------------
def hash_join_indices(left_keys, right_keys, join_type: str = "inner"):
    """(left rows, right rows or None) in left-row order, matches of a left row in right-row order; right is None (a null
    index) for the unmatched rows of "left outer"; "left semi" / "left anti" return (left rows, None)."""
    lrows = list(Grouper([k.type for k in left_keys])._rows(left_keys))
    rrows = list(Grouper([k.type for k in right_keys])._rows(right_keys))
    table = {}
    for j, row in enumerate(rrows):
        if any(v is None for v in row):
            continue
        table.setdefault(row, []).append(j)
    left, right = [], []
    for i, row in enumerate(lrows):
        hits = [] if any(v is None for v in row) else table.get(row, [])
        if join_type == "inner":
            left += [i] * len(hits)
            right += hits
        elif join_type in ("left outer", "full outer"):
            left += [i] * max(1, len(hits))
            right += hits if hits else [None]
        elif join_type == "left semi":
            left += [i] if hits else []
        elif join_type == "left anti":
            left += [] if hits else [i]
        else:
            raise ValueError(join_type)
    if join_type == "full outer":  # then the right rows nobody matched (null key, or no equal left key), in row order
        hit_right = {j for j in right if j is not None}
        lonely = [j for j in range(len(rrows)) if j not in hit_right]
        left += [None] * len(lonely)
        right += lonely
    li = pa.array(left, pa.uint32())
    if join_type in ("left semi", "left anti"):
        return li, None
    return li, pa.array(right, pa.uint32())
