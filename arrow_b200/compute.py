"""Host-side mirror of the reference's function API for the hot path.

Same names, argument meaning and error behaviour as arrow::compute::CallFunction
(cpp/src/arrow/compute/exec.cc:1362-1390) / pyarrow.compute, but operands are
DeviceArray and every kernel is a C-ABI call into libarrow_b200.so.  The dispatch rules
reproduced here are the reference's:
  * arithmetic / compare: exact match, else promote all operands to CommonNumeric
    (kernels/codegen_internal.cc:166-218) with an implicit safe cast
    (ArithmeticFunction::DispatchBest kernels/scalar_arithmetic.cc:734-781,
     CompareFunction::DispatchBest kernels/scalar_compare.cc:340-366,
     FunctionExecutorImpl::Execute function.cc:242-250),
  * filter / take / sort_indices meta-functions unwrap to array_* kernels
    (kernels/vector_selection_filter_internal.cc:1043-1072, vector_selection_take_internal.cc:660-701,
     kernels/vector_sort.cc:856-924).
"""
from __future__ import annotations

import builtins
import ctypes as C
import re
from typing import Optional, Sequence, Union

import numpy as np
import pyarrow as pa

from . import _cabi as cabi
from .device import _NUMERIC as _NUMERIC_TYPES
from .device import Context, DeviceArray, NativeHandle, arrow_type, check, type_id

Operand = Union[DeviceArray, pa.Scalar, int, float, bool, None]

_NUMERIC_IDS = (cabi.UINT8, cabi.INT8, cabi.UINT16, cabi.INT16, cabi.UINT32, cabi.INT32, cabi.UINT64,
                cabi.INT64, cabi.FLOAT, cabi.DOUBLE)
_SIGNED = {cabi.INT8: 8, cabi.INT16: 16, cabi.INT32: 32, cabi.INT64: 64}
_UNSIGNED = {cabi.UINT8: 8, cabi.UINT16: 16, cabi.UINT32: 32, cabi.UINT64: 64}
_NP = {cabi.INT8: np.int8, cabi.UINT8: np.uint8, cabi.INT16: np.int16, cabi.UINT16: np.uint16,
       cabi.INT32: np.int32, cabi.UINT32: np.uint32, cabi.INT64: np.int64, cabi.UINT64: np.uint64,
       cabi.FLOAT: np.float32, cabi.DOUBLE: np.float64}


def _ctx(*args) -> Context:
    for a in args:
        if isinstance(a, DeviceArray):
            return a.ctx
    return Context.get()


def _list(ctx: Context, offsets: cabi.B2Array, child: DeviceArray, value_type: pa.DataType) -> DeviceArray:
    """list<value_type> from the int32 offsets an entry point allocated and its child"""
    return DeviceArray(ctx, pa.list_(value_type), offsets.length - 1, 0, 0, [None, ctx.adopt(offsets.data, 4 * offsets.length)],
                       children=[child])


def _out(ctx: Context, c: cabi.B2Array, type: pa.DataType, dictionary=None) -> DeviceArray:
    return DeviceArray._from_c(ctx, c, type, dictionary)


def _call(ctx: Context, fn: str, out_type: Optional[pa.DataType], *args, handle=None, dictionary=None) -> DeviceArray:
    """ctx.lib.<fn>(handle, *args, B2Array* out, stream), `handle` being the context's unless given: its output as a
    DeviceArray of out_type, or of the type the entry point reports when out_type is None."""
    cout = cabi.B2Array()
    check(getattr(ctx.lib, fn)(ctx.handle if handle is None else handle, *args, C.byref(cout), ctx.stream))
    return _out(ctx, cout, arrow_type(cout.type) if out_type is None else out_type, dictionary)


# every spelling an enum argument accepts, with its code
_NULL_SELECTION = {"drop": 0, 0: 0, None: 0, "emit_null": 1, 1: 1}
_ORDER = {"ascending": 0, 0: 0, "descending": 1, 1: 1}
_PLACEMENT = {"at_start": 0, 0: 0, "at_end": 1, 1: 1}
_NULL_ENCODING = {"mask": 0, 0: 0, "encode": 1, 1: 1}
_COUNT_MODE = {"only_valid": 0, "only_null": 1, "all": 2}


def _enum(value, codes: dict, what: str) -> int:
    for spelling, code in codes.items():
        if value == spelling:
            return code
    raise ValueError(f'"{value}" is not a valid {what}')


# ------------------------------------------------------------------------------------
# dispatch helpers
# ------------------------------------------------------------------------------------
def common_numeric(ids: Sequence[int]) -> int:
    """CommonNumeric (kernels/codegen_internal.cc:166-218)."""
    for i in ids:
        if i not in _NUMERIC_IDS:
            raise pa.ArrowNotImplementedError("Function has no kernel matching input types")
    if cabi.DOUBLE in ids:
        return cabi.DOUBLE
    if cabi.FLOAT in ids:
        return cabi.FLOAT
    ms = builtins.max([_SIGNED[i] for i in ids if i in _SIGNED], default=0)
    mu = builtins.max([_UNSIGNED[i] for i in ids if i in _UNSIGNED], default=0)
    if ms == 0:
        return {8: cabi.UINT8, 16: cabi.UINT16, 32: cabi.UINT32}.get(mu, cabi.UINT64)
    if ms <= mu:
        ms = 1 << (mu + 1 - 1).bit_length()  # NextPower2(mu + 1)
    return {8: cabi.INT8, 16: cabi.INT16, 32: cabi.INT32}.get(ms, cabi.INT64)


def _require_numeric(t: pa.DataType) -> None:
    """Only the ten genuinely numeric Arrow types reach the numeric kernels.  Temporal / dictionary /
    other logical types share an integer STORAGE with them but not their semantics (the reference
    rescales units in casts, kernels/scalar_cast_temporal.cc, and dispatches timestamp/duration
    arithmetic to dedicated kernels, kernels/scalar_arithmetic.cc:1480-1529): refuse rather than
    compute on raw storage."""
    if t not in _NUMERIC_TYPES:
        raise pa.ArrowNotImplementedError(f"Function has no kernel matching input types ({t}) on arrow_b200 device arrays")


_BINARY_TYPES = {pa.string(), pa.binary(), pa.large_string(), pa.large_binary()}


def _require_sort_key(t: pa.DataType) -> None:
    """Sort keys are the numeric types or the four base-binary types (ordered by their bytes, unsigned,
    a proper prefix first: ArrayCompareSorter, kernels/vector_array_sort.cc:144-178)."""
    if t not in _BINARY_TYPES:
        _require_numeric(t)


def _as_scalar(x) -> pa.Scalar:
    if isinstance(x, pa.Scalar):
        return x
    return pa.scalar(x)


def _safe_int_range(src: int, dst: int):
    """The values of integer type `src` that a safe cast to `dst` admits, as (lo, hi) in `src`: the intersection of the
    two ranges for an integer target (GetSafeMinMax, util/int_util.cc), and +-2^24 / +-2^53 for a float target
    that cannot hold every `src` value exactly (kernels/scalar_cast_numeric.cc:214-279, the bound b2_cast_numeric
    applies to arrays)."""
    info = np.iinfo(_NP[src])
    lo, hi = int(info.min), int(info.max)
    if dst in _SIGNED or dst in _UNSIGNED:
        dinfo = np.iinfo(_NP[dst])
        return builtins.max(lo, int(dinfo.min)), builtins.min(hi, int(dinfo.max))
    bits = _SIGNED.get(src) or _UNSIGNED[src]
    if bits < 32 or (bits == 32 and dst == cabi.DOUBLE):
        return lo, hi
    limit = 1 << (24 if dst == cabi.FLOAT else 53)
    return builtins.max(lo, -limit if src in _SIGNED else 0), builtins.min(hi, limit)


def _scalar_to(s: pa.Scalar, tid: int) -> cabi.B2Scalar:
    """Implicit safe cast of a host scalar to the dispatched type (done on the host: it is
    argument preparation, one value), with the errors and texts of the reference's safe cast.
    A scalar that already has the type keeps its exact bits (a signalling NaN's included)."""
    out = cabi.B2Scalar()
    out.type = tid
    out.is_valid = 1 if s.is_valid else 0
    out.bits = 0
    if s.is_valid and tid == cabi.BOOL:
        out.bits = int(s.as_py())
    elif s.is_valid:
        src = type_id(s.type)
        dt = _NP[tid]
        if src == tid:
            raw = pa.array([s], s.type).buffers()[1].to_pybytes()[:np.dtype(dt).itemsize]
            out.bits = int.from_bytes(raw, "little")
            return out
        v = s.as_py()
        if isinstance(v, float):
            if np.issubdtype(dt, np.integer):  # unreachable from CommonNumeric (a float operand makes a float type)
                info = np.iinfo(dt)
                if not (np.isfinite(v) and v == int(v) and info.min <= int(v) <= info.max):
                    raise pa.ArrowInvalid(f"Float value {v:f} was truncated converting to {arrow_type(tid)}")
                v = int(v)
            arr = np.array([v], dtype=dt)  # float32 -> float64 is exact
        else:
            lo, hi = _safe_int_range(src, tid)
            if not lo <= v <= hi:
                raise pa.ArrowInvalid(f"Integer value {v} not in range: {lo} to {hi}")
            arr = np.array([v], dtype=dt)  # exact: inside the safe range every value is representable
        out.bits = int(np.frombuffer(arr.tobytes().ljust(8, b"\0"), dtype=np.uint64)[0])
    return out


def _numeric_operands(*xs):
    """xs as numeric DeviceArrays / pa.Scalars, checked one after the other, and the type id they dispatch to: theirs
    when they agree, else their CommonNumeric."""
    ops = []
    for x in xs:
        x = x if isinstance(x, DeviceArray) else _as_scalar(x)
        if pa.types.is_null(x.type):
            raise pa.ArrowNotImplementedError("null-typed scalar operands are not supported")
        _require_numeric(x.type)
        ops.append(x)
    ids = [type_id(o.type) for o in ops]
    return ops, (ids[0] if ids[0] == ids[1] else common_numeric(ids))


def _bool_operand(x):
    """x as a boolean DeviceArray or a boolean / null-typed pa.Scalar"""
    x = x if isinstance(x, DeviceArray) else _as_scalar(x)
    if not (pa.types.is_boolean(x.type) or pa.types.is_null(x.type)):
        raise pa.ArrowNotImplementedError(f"Function has no kernel matching input types ({x.type})")
    return x


def _value(x: Union[DeviceArray, pa.Scalar], tid: int, keep: list) -> cabi.B2Value:
    """Operand x as a B2Value of type tid, after the implicit safe cast: on the device for an array, by _scalar_to for a
    scalar.  What the value points to is appended to `keep`, which must outlive the call."""
    v = cabi.B2Value()
    if isinstance(x, DeviceArray):
        if type_id(x.type) != tid:
            x = cast(x, arrow_type(tid))
        c = x._c()
        keep.append((x, c))
        v.array = C.pointer(c)
    else:
        sc = _scalar_to(x, tid)
        keep.append(sc)
        v.scalar = C.pointer(sc)
    return v


def _prepare_binary(left: Operand, right: Operand):
    ctx = _ctx(left, right)
    ops, tid = _numeric_operands(left, right)
    if not any(isinstance(o, DeviceArray) for o in ops):
        raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
    keep = []
    return ctx, tid, [_value(o, tid, keep) for o in ops], keep


# ------------------------------------------------------------------------------------
# scalar kernels
# ------------------------------------------------------------------------------------
def cast(arr: DeviceArray, target_type=None, safe: Optional[bool] = None, options=None) -> DeviceArray:
    """pyarrow.compute.cast / CastMetaFunction (compute/cast.cc:78-127)."""
    allow_int_overflow = allow_float_truncate = False
    if options is not None:
        target_type = options.target_type if target_type is None else target_type
        allow_int_overflow = bool(options.allow_int_overflow)
        allow_float_truncate = bool(options.allow_float_truncate)
    if safe is False:
        allow_int_overflow = allow_float_truncate = True
    target_type = pa.lib.ensure_type(target_type)
    if arr.type == target_type:
        return arr
    # logical types (timestamp/date/time/duration/dictionary) have numeric STORAGE ids but unit / index
    # semantics the numeric cast kernel does not implement: only exact numeric types pass
    if arr.type not in _NUMERIC_TYPES or target_type not in _NUMERIC_TYPES:
        raise pa.ArrowNotImplementedError(
            f"Unsupported cast from {arr.type} to {target_type} using function cast_{target_type}")
    src, dst = type_id(arr.type), type_id(target_type)
    if src not in _NUMERIC_IDS or dst not in _NUMERIC_IDS:
        raise pa.ArrowNotImplementedError(
            f"Unsupported cast from {arr.type} to {target_type} using function cast_{target_type}")
    opt = cabi.B2CastOptions(dst, int(allow_int_overflow), int(allow_float_truncate), 0)
    return _call(arr.ctx, "b2_cast_numeric", target_type, C.byref(arr._c()), C.byref(opt))


def _arith(name: str, left: Operand, right: Operand) -> DeviceArray:
    ctx, tid, vals, keep = _prepare_binary(left, right)
    return _call(ctx, "b2_binary_arith", arrow_type(tid), cabi.ARITH_OPS[name], C.byref(vals[0]), C.byref(vals[1]))


def _binary_like(x):
    """x as a binary-like DeviceArray or pa.Scalar (str / bytes become utf8 / binary scalars), else None"""
    if isinstance(x, DeviceArray):
        return x if x.type in _BINARY_TYPES else None
    if isinstance(x, (str, bytes)):
        return pa.scalar(x)
    if isinstance(x, pa.Scalar) and x.type in _BINARY_TYPES:
        return x
    return None


def _type_name(x) -> str:
    if isinstance(x, (DeviceArray, pa.Scalar)):
        return str(x.type)
    return str(_as_scalar(x).type)


_FLIPPED = {"equal": "equal", "not_equal": "not_equal", "greater": "less", "greater_equal": "less_equal",
            "less": "greater", "less_equal": "greater_equal"}


def _compare_binary(name: str, left, right) -> DeviceArray:
    """equal ... less_equal over utf8 / large_utf8 / binary / large_binary (scalar_compare.cc:42-72,431-433): unsigned
    bytewise order, a proper prefix first.  Any pair of the four types is compared as it is (CompareFunction::DispatchBest
    would cast both to CommonBinary; the bytes compared are the same).  A scalar-array call is the array-scalar call
    with the operator flipped."""
    lb, rb = _binary_like(left), _binary_like(right)
    if lb is None or rb is None:
        raise pa.ArrowNotImplementedError(
            f"Function '{name}' has no kernel matching input types ({_type_name(left)}, {_type_name(right)})")
    if not isinstance(lb, DeviceArray):
        if not isinstance(rb, DeviceArray):
            raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
        lb, rb, name = rb, lb, _FLIPPED[name]
    if isinstance(rb, DeviceArray):
        right_args = (C.byref(rb._c()), None, 0, 1)
    else:
        raw = rb.as_buffer().to_pybytes() if rb.is_valid else b""
        right_args = (None, raw, len(raw), int(rb.is_valid))
    return _call(lb.ctx, "b2_compare_binary", pa.bool_(), cabi.COMPARE_OPS[name], C.byref(lb._c()), *right_args)


def _compare(name: str, left: Operand, right: Operand) -> DeviceArray:
    if _binary_like(left) is not None or _binary_like(right) is not None:
        return _compare_binary(name, left, right)
    ctx, tid, vals, keep = _prepare_binary(left, right)
    return _call(ctx, "b2_compare", pa.bool_(), cabi.COMPARE_OPS[name], C.byref(vals[0]), C.byref(vals[1]))


def add(x, y): return _arith("add", x, y)
def subtract(x, y): return _arith("subtract", x, y)
def multiply(x, y): return _arith("multiply", x, y)
def divide(x, y): return _arith("divide", x, y)
def add_checked(x, y): return _arith("add_checked", x, y)
def subtract_checked(x, y): return _arith("subtract_checked", x, y)
def multiply_checked(x, y): return _arith("multiply_checked", x, y)
def divide_checked(x, y): return _arith("divide_checked", x, y)
def equal(x, y): return _compare("equal", x, y)
def not_equal(x, y): return _compare("not_equal", x, y)
def greater(x, y): return _compare("greater", x, y)
def greater_equal(x, y): return _compare("greater_equal", x, y)
def less(x, y): return _compare("less", x, y)
def less_equal(x, y): return _compare("less_equal", x, y)


# ------------------------------------------------------------------------------------
# boolean logic + validity predicates (kernels/scalar_boolean.cc, kernels/scalar_validity.cc)
# ------------------------------------------------------------------------------------
def _boolean(name: str, left, right=None) -> DeviceArray:
    ctx = _ctx(left, right)
    keep = []
    lv = _value(_bool_operand(left), cabi.BOOL, keep)
    rv = C.byref(_value(_bool_operand(right), cabi.BOOL, keep)) if name != "invert" else None
    return _call(ctx, "b2_boolean", pa.bool_(), cabi.BOOLEAN_OPS[name], C.byref(lv), rv)


def and_(x, y): return _boolean("and", x, y)
def or_(x, y): return _boolean("or", x, y)
def xor(x, y): return _boolean("xor", x, y)
def and_not(x, y): return _boolean("and_not", x, y)
def and_kleene(x, y): return _boolean("and_kleene", x, y)
def or_kleene(x, y): return _boolean("or_kleene", x, y)
def and_not_kleene(x, y): return _boolean("and_not_kleene", x, y)
def invert(x): return _boolean("invert", x)


def _validity(name: str, arr: DeviceArray, nan_is_null: bool = False) -> DeviceArray:
    return _call(arr.ctx, "b2_validity", pa.bool_(), cabi.VALIDITY_OPS[name], C.byref(arr._c()), int(bool(nan_is_null)))


def is_valid(x): return _validity("is_valid", x)
def is_null(x, nan_is_null=False): return _validity("is_null", x, nan_is_null)
def true_unless_null(x): return _validity("true_unless_null", x)
def is_nan(x): return _validity("is_nan", x)


def if_else(cond, left, right) -> DeviceArray:
    """if_else (kernels/scalar_if_else.cc:62-520): cond ? left : right, null where cond or the chosen side is null.
    cond: boolean DeviceArray or scalar; left / right: DeviceArrays or scalars, numerics promoted to their common type
    like the reference's DispatchBest (scalar_if_else.cc:1227-1266), or both boolean."""
    ctx = _ctx(cond, left, right)
    keep = []
    cv = _value(_bool_operand(cond), cabi.BOOL, keep)
    sides = [x if isinstance(x, DeviceArray) else _as_scalar(x) for x in (left, right)]
    if all(pa.types.is_boolean(x.type) or pa.types.is_null(x.type) for x in sides):
        tid = cabi.BOOL
    else:
        sides, tid = _numeric_operands(*sides)
    vals = [_value(x, tid, keep) for x in sides]
    return _call(ctx, "b2_if_else", arrow_type(tid), C.byref(cv), C.byref(vals[0]), C.byref(vals[1]))


# ------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------
def filter(values: DeviceArray, mask: DeviceArray, null_selection_behavior="drop") -> DeviceArray:
    """pyarrow.compute.filter / array_filter (kernels/vector_selection_filter_internal.cc:1043-1072)."""
    if not pa.types.is_boolean(mask.type):
        raise pa.ArrowNotImplementedError(
            f"Function 'array_filter' has no kernel matching input types ({values.type}, {mask.type})")
    if len(values) != len(mask):  # raised by the reference's VectorExecutor before the kernel runs
        raise pa.ArrowInvalid("Arguments for execution of vector kernel function 'array_filter' must all be the same length")
    return _call(values.ctx, "b2_filter", values.type, C.byref(values._c()), C.byref(mask._c()),
                 _enum(null_selection_behavior, _NULL_SELECTION, "null selection behavior"), dictionary=values.dictionary)


def array_filter(values, mask, null_selection_behavior="drop"):
    return filter(values, mask, null_selection_behavior)


def filter_output_size(mask: DeviceArray, null_selection_behavior="drop") -> int:
    ctx = mask.ctx
    n = C.c_int64()
    cm = mask._c()
    behavior = _enum(null_selection_behavior, _NULL_SELECTION, "null selection behavior")
    check(ctx.lib.b2_filter_output_size(ctx.handle, C.byref(cm), behavior, C.byref(n), ctx.stream))
    return n.value


def take_indices_from_filter(mask: DeviceArray, null_selection_behavior="drop") -> DeviceArray:
    """GetTakeIndices (kernels/vector_selection_take_internal.cc:298-305)."""
    return _call(mask.ctx, "b2_filter_indices", None, C.byref(mask._c()),
                 _enum(null_selection_behavior, _NULL_SELECTION, "null selection behavior"))


def take(values: DeviceArray, indices: DeviceArray, boundscheck: bool = True) -> DeviceArray:
    """pyarrow.compute.take / array_take (kernels/vector_selection_take_internal.cc:660-701)."""
    if not pa.types.is_integer(indices.type):
        raise pa.ArrowNotImplementedError(
            f"Function 'array_take' has no kernel matching input types ({values.type}, {indices.type})")
    return _call(values.ctx, "b2_take", values.type, C.byref(values._c()), C.byref(indices._c()), int(bool(boundscheck)),
                 dictionary=values.dictionary)


def take_cast_arith(values: DeviceArray, indices: DeviceArray, target_type, op: str, other) -> DeviceArray:
    """Fused `op(cast(take(values, indices), target_type, safe=False), other)` -- one kernel instead of three
    (b2_take_cast_arith; the reference evaluates the same Expression kernel by kernel, compute/expression.cc:722-797).
    Falls back to the three calls for operand shapes the fused kernel does not cover."""
    target_type = pa.lib.ensure_type(target_type)
    fusable = (values.type in (pa.float64(), pa.float32(), pa.int64(), pa.int32()) and target_type in (pa.float32(), pa.float64())
               and indices.type in (pa.int32(), pa.uint32(), pa.int64(), pa.uint64()) and op in ("add", "subtract", "multiply")
               and isinstance(other, DeviceArray) and other.type == target_type and len(other) == len(indices))
    if not fusable:
        return _arith(op, cast(take(values, indices), target_type, safe=False), other)
    keep = []
    ov = _value(other, type_id(target_type), keep)
    return _call(values.ctx, "b2_take_cast_arith", target_type, C.byref(values._c()), C.byref(indices._c()),
                 type_id(target_type), cabi.ARITH_OPS[op], C.byref(ov))


def array_take(values, indices, boundscheck=True):
    return take(values, indices, boundscheck)


# ------------------------------------------------------------------------------------
# sort
# ------------------------------------------------------------------------------------
def array_sort_indices(arr: DeviceArray, order="ascending", null_placement="at_end") -> DeviceArray:
    """array_sort_indices (kernels/vector_array_sort.cc:524-540): stable argsort -> uint64."""
    return _call(arr.ctx, "b2_sort_indices", pa.uint64(), C.byref(arr._c()), _enum(order, _ORDER, "order"),
                 _enum(null_placement, _PLACEMENT, "null placement"))


def sort_payload(arr: DeviceArray, payload: DeviceArray, order="ascending", null_placement="at_end") -> DeviceArray:
    """stable sort of `arr` where row i carries payload[i] (uint32) instead of i: returns the payloads in sorted order
    (uint64) -- array_sort_indices followed by take(payload, indices), in the radix passes themselves"""
    return _call(arr.ctx, "b2_sort_payload", pa.uint64(), C.byref(arr._c()), C.byref(payload._c()),
                 _enum(order, _ORDER, "order"), _enum(null_placement, _PLACEMENT, "null placement"))


def sort_indices(arr, sort_keys=None, null_placement="at_end", order=None) -> DeviceArray:
    """sort_indices meta function (kernels/vector_sort.cc:850-1027): on one array, or -- given a mapping
    {name: DeviceArray} (a record batch / table of device columns) and sort_keys = [(name, order), ...] -- the
    multi-key sort: ordered by the first key, ties by the next, stable (b2_sort_indices_multi)."""
    if isinstance(arr, dict):
        if not sort_keys:
            raise pa.ArrowInvalid("Must specify one or more sort keys")
        cols, orders = [], []
        for k in sort_keys:
            name, o = (k[0], k[1]) if isinstance(k, (tuple, list)) else (k, "ascending")
            if name not in arr:
                raise pa.ArrowInvalid(f"No match for FieldRef.Name({name})")
            _require_sort_key(arr[name].type)
            cols.append(arr[name])
            orders.append(_enum(o, _ORDER, "order"))
        cks = (cabi.B2Array * len(cols))(*[c._c() for c in cols])
        cor = (C.c_int32 * len(cols))(*orders)
        return _call(cols[0].ctx, "b2_sort_indices_multi", pa.uint64(), cks, len(cols), cor,
                     _enum(null_placement, _PLACEMENT, "null placement"))
    o = "ascending"
    if sort_keys:
        o = sort_keys[0][1] if isinstance(sort_keys[0], (tuple, list)) else sort_keys[0]
    if order is not None:
        o = order
    return array_sort_indices(arr, o, null_placement)


def select_k_unstable(arr: DeviceArray, k: int, sort_keys=None, null_placement="at_end") -> DeviceArray:
    """select_k_unstable (kernels/vector_select_k.cc:157-232, SelectKOptions api_vector.h:178-214) on one array: the
    indices of the first k rows in sort order; sort_keys = [(ignored name, order)] as in the reference.  Ties come out in
    row order (= sort_indices(...)[:k]), one of the answers the reference's unstable selection may give."""
    if k < 0:
        raise pa.ArrowInvalid(f"select_k_unstable requires a nonnegative `k`, got {k}")
    o = "ascending"
    if sort_keys:
        if len(sort_keys) != 1:
            raise pa.ArrowNotImplementedError("arrow_b200 select_k_unstable: one sort key (use sort_indices for several)")
        o = sort_keys[0][1] if isinstance(sort_keys[0], (tuple, list)) else "ascending"
    _require_sort_key(arr.type)
    return _call(arr.ctx, "b2_select_k", pa.uint64(), C.byref(arr._c()), int(k), _enum(o, _ORDER, "order"),
                 _enum(null_placement, _PLACEMENT, "null placement"))


# ------------------------------------------------------------------------------------
# ungrouped aggregates (kernels/aggregate_basic.cc, aggregate_basic.inc.cc)
# ------------------------------------------------------------------------------------
def _reduce(arr: DeviceArray) -> "cabi.B2ReduceResult":
    _require_numeric(arr.type)
    ctx = arr.ctx
    ca, r = arr._c(), cabi.B2ReduceResult()
    check(ctx.lib.b2_reduce(ctx.handle, C.byref(ca), C.byref(r), ctx.stream))
    return r


def _from_bits(bits: int, t: pa.DataType):
    raw = np.array([bits], dtype=np.uint64)
    if pa.types.is_floating(t):
        return raw.view(np.float64)[0]
    return raw.view(np.int64)[0] if pa.types.is_signed_integer(t) else raw[0]


def _acc_type(t: pa.DataType) -> pa.DataType:
    if pa.types.is_floating(t):
        return pa.float64()
    return pa.int64() if pa.types.is_signed_integer(t) else pa.uint64()


def sum(arr: DeviceArray, skip_nulls: bool = True, min_count: int = 1) -> pa.Scalar:  # noqa: A001
    """sum (SumImpl::Finalize, aggregate_basic.inc.cc:95-103): null if a null was seen and
    !skip_nulls, or fewer than min_count valid values; accumulator = int64 / uint64 / double."""
    r, out_t = _reduce(arr), _acc_type(arr.type)
    if (not skip_nulls and r.null_count > 0) or r.count < min_count:
        return pa.scalar(None, out_t)
    return pa.scalar(_from_bits(r.sum_bits, out_t).item(), out_t)


def mean(arr: DeviceArray, skip_nulls: bool = True, min_count: int = 1) -> pa.Scalar:
    """mean (MeanImpl, aggregate_basic.inc.cc:263-283): the sum is accumulated in double, then / count."""
    r = _reduce(arr)
    if (not skip_nulls and r.null_count > 0) or r.count < min_count:
        return pa.scalar(None, pa.float64())
    with np.errstate(invalid="ignore", divide="ignore"):  # no valid value and min_count == 0: 0/0 = NaN like the reference
        return pa.scalar(float(_from_bits(r.dsum_bits, pa.float64()) / np.float64(r.count)), pa.float64())


def min_max(arr: DeviceArray, skip_nulls: bool = True, min_count: int = 1) -> pa.Scalar:
    """min_max (MinMaxImpl::Finalize, aggregate_basic.inc.cc:834-853): struct<min, max> of the input
    type; min_count is at least 1 (:783)."""
    r, t = _reduce(arr), arr.type
    st = pa.struct([("min", t), ("max", t)])
    if (r.null_count > 0 and not skip_nulls) or r.count < builtins.max(1, min_count):
        return pa.scalar({"min": None, "max": None}, st)
    wide = _acc_type(t)
    lo, hi = _from_bits(r.min_bits, wide), _from_bits(r.max_bits, wide)
    nt = np.dtype(t.to_pandas_dtype()).type
    return pa.scalar({"min": nt(lo).item(), "max": nt(hi).item()}, st)


def min(arr: DeviceArray, skip_nulls: bool = True, min_count: int = 1) -> pa.Scalar:  # noqa: A001
    return min_max(arr, skip_nulls, min_count)["min"]


def max(arr: DeviceArray, skip_nulls: bool = True, min_count: int = 1) -> pa.Scalar:  # noqa: A001
    return min_max(arr, skip_nulls, min_count)["max"]


def count(arr: DeviceArray, mode: str = "only_valid") -> pa.Scalar:
    """count (CountImpl, aggregate_basic.cc:98-130; CountOptions api_aggregate.h:64-78)."""
    ctx = arr.ctx
    nulls = arr.null_count
    if nulls < 0:  # unknown after slicing: count the validity bits on the device
        out = C.c_int64()
        check(ctx.lib.b2_bitmap_count(ctx.handle, arr.buffers[0].ptr, arr.offset, arr.length, C.byref(out), ctx.stream))
        nulls = arr.length - out.value
    return pa.scalar((arr.length - nulls, nulls, arr.length)[_enum(mode, _COUNT_MODE, "count mode")], pa.int64())


# ------------------------------------------------------------------------------------
# unique / value_counts / dictionary_encode (kernels/vector_hash.cc:782-830)
# ------------------------------------------------------------------------------------
def _vector_hash(arr: DeviceArray, null_encoding: int, want_indices: bool, want_counts: bool):
    ctx = arr.ctx
    ca, ci, cd, cc = arr._c(), cabi.B2Array(), cabi.B2Array(), cabi.B2Array()
    check(ctx.lib.b2_vector_hash(ctx.handle, C.byref(ca), null_encoding, C.byref(ci) if want_indices else None,
                                 C.byref(cd), C.byref(cc) if want_counts else None, ctx.stream))
    dictionary = _out(ctx, cd, arr.type)
    indices = _out(ctx, ci, pa.dictionary(pa.int32(), arr.type), dictionary) if want_indices else None
    counts = _out(ctx, cc, pa.int64()) if want_counts else None
    return indices, dictionary, counts


def unique(arr: DeviceArray) -> DeviceArray:
    """unique: distinct values in first-occurrence order, null included (vector_hash.cc:65-97,791)."""
    return _vector_hash(arr, 1, False, False)[1]


def value_counts(arr: DeviceArray):
    """value_counts: (values, counts) = the two fields of the reference's struct result
    (vector_hash.cc:101-168,634,807); `to_struct` below assembles the StructArray on the host."""
    _, values, counts = _vector_hash(arr, 1, False, True)
    return values, counts


def value_counts_to_struct(values: DeviceArray, counts: DeviceArray) -> pa.StructArray:
    return pa.StructArray.from_arrays([values.to_arrow(), counts.to_arrow()], names=["values", "counts"])


def count_distinct(arr: DeviceArray, mode: str = "only_valid") -> pa.Scalar:
    """count_distinct (CountDistinctImpl, kernels/aggregate_basic.cc:141-230; CountOptions api_aggregate.h:64-78): the size of
    the memo table = the number of uniques, with the null entry counted under only_null / all."""
    u = unique(arr)
    has_null = 1 if u.null_count > 0 else 0
    return pa.scalar((len(u) - has_null, has_null, len(u))[_enum(mode, _COUNT_MODE, "count mode")], pa.int64())


def dictionary_encode(arr: DeviceArray, null_encoding="mask") -> DeviceArray:
    """dictionary_encode: int32 indices + dictionary (vector_hash.cc:173-232,826;
    DictionaryEncodeOptions api_vector.h:66-82)."""
    return _vector_hash(arr, _enum(null_encoding, _NULL_ENCODING, "null encoding behavior"), True, False)[0]


# ------------------------------------------------------------------------------------
# is_in / index_in (kernels/scalar_set_lookup.cc; SetLookupOptions compute/api_scalar.h:279-324)
# ------------------------------------------------------------------------------------
NULL_MATCHING = {"match": 0, "skip": 1, "emit_null": 2, "inconclusive": 3}
_SET_LOOKUP_TYPES = set(_NUMERIC_TYPES) | _BINARY_TYPES | {pa.bool_()}
_STRING_TYPES = {pa.string(), pa.large_string()}


def _null_matching(skip_nulls, null_matching_behavior) -> int:
    """GetNullMatchingBehavior (api_scalar.cc:604-612): skip_nulls=True is SKIP; otherwise null_matching_behavior,
    MATCH when it is not given."""
    if skip_nulls:
        return NULL_MATCHING["skip"]
    if null_matching_behavior is None:
        return NULL_MATCHING["match"]
    return _enum(null_matching_behavior, NULL_MATCHING, "null matching behavior")


def _lookup_table(ctx: Context, value_set: cabi.B2Array, null_matching: int) -> NativeHandle:
    return NativeHandle(ctx, "b2_set_lookup_destroy",
                        lambda h: ctx.lib.b2_set_lookup_create(ctx.handle, C.byref(value_set), null_matching, h, ctx.stream))


def _set_lookup_casts(values_type: pa.DataType, value_set: DeviceArray):
    """InitStateVisitor::GetResult (scalar_set_lookup.cc:213-258): the value set cast to the values' type (safe), or, when
    that cast fails, the values cast to the value set's type at exec time.  Returns (value set, type to cast values to)."""
    vt, st = values_type, value_set.type
    if (vt in _STRING_TYPES and st not in _BINARY_TYPES) or (st in _STRING_TYPES and vt not in _BINARY_TYPES):
        raise pa.ArrowTypeError(f"Array type doesn't match type of values set: {vt} vs {st}")
    if vt == st:
        return value_set, None
    if vt not in _NUMERIC_TYPES or st not in _NUMERIC_TYPES:
        raise pa.ArrowNotImplementedError(f"arrow_b200 is_in / index_in: no device cast between {st} and {vt}")
    try:
        return cast(value_set, vt, safe=True), None
    except pa.ArrowInvalid:
        return value_set, st  # every numeric type casts to every other (CanCast)


def _set_lookup(values, value_set, skip_nulls, null_matching_behavior, index: bool):
    if value_set is None:
        raise pa.ArrowInvalid("Attempted to call a set lookup function without SetLookupOptions")
    chunks = [values] if isinstance(values, DeviceArray) else list(values)
    ctx = chunks[0].ctx if chunks else _ctx(value_set)
    vt = chunks[0].type if chunks else value_set.type
    if vt not in _SET_LOOKUP_TYPES or any(c.type != vt for c in chunks):
        raise pa.ArrowNotImplementedError(f"Function has no kernel matching input types ({vt}) on arrow_b200 device arrays")
    if isinstance(value_set, pa.ChunkedArray):
        value_set = pa.concat_arrays(value_set.chunks) if value_set.num_chunks else pa.array([], value_set.type)
    if isinstance(value_set, pa.Array):
        value_set = DeviceArray.from_arrow(value_set, ctx)
    if value_set.type not in _SET_LOOKUP_TYPES:
        raise pa.ArrowNotImplementedError(f"arrow_b200 is_in / index_in: value set type {value_set.type} is not supported on device")
    value_set, cast_to = _set_lookup_casts(vt, value_set)
    nm = _null_matching(skip_nulls, null_matching_behavior)
    outs = []
    with _lookup_table(ctx, value_set._c(), nm) as table:
        for c in chunks:  # the table is built once and probed per chunk
            if cast_to is not None:
                c = cast(c, cast_to, safe=True)
            outs.append(_call(ctx, "b2_index_in" if index else "b2_is_in", pa.int32() if index else pa.bool_(),
                              C.byref(c._c()), handle=table.handle))
    return outs[0] if isinstance(values, DeviceArray) else outs


def is_in(values, value_set=None, skip_nulls: bool = False, null_matching_behavior: Optional[str] = None):
    """is_in (ExecIsIn, scalar_set_lookup.cc:398-545): whether each value is in value_set.  values: a DeviceArray, or a
    list of chunks (one result per chunk); value_set: a pyarrow Array / ChunkedArray (uploaded) or a DeviceArray.
    null_matching_behavior: "match" (default), "skip", "emit_null" or "inconclusive"; skip_nulls=True is "skip"."""
    return _set_lookup(values, value_set, skip_nulls, null_matching_behavior, False)


def index_in(values, value_set=None, skip_nulls: bool = False, null_matching_behavior: Optional[str] = None):
    """index_in (ExecIndexIn, scalar_set_lookup.cc:271-396): the int32 position of each value's first occurrence in
    value_set, null where there is none; arguments as for is_in."""
    return _set_lookup(values, value_set, skip_nulls, null_matching_behavior, True)


def set_lookup_table(value_set: DeviceArray, null_matching_behavior: str = "match"):
    """(table bytes, staged in shared memory) of the table b2_set_lookup_create builds for value_set."""
    ctx, nbytes, shared = value_set.ctx, C.c_int64(), C.c_int32()
    with _lookup_table(ctx, value_set._c(), NULL_MATCHING[null_matching_behavior]) as table:
        check(ctx.lib.b2_set_lookup_table(table.handle, C.byref(nbytes), C.byref(shared)))
    return nbytes.value, bool(shared.value)


# ------------------------------------------------------------------------------------
# match_substring / starts_with / ends_with / match_like (kernels/scalar_string_ascii.cc:1221-1307,1456-1588;
# MatchSubstringOptions compute/api_scalar.h)
# ------------------------------------------------------------------------------------
def _string_match(name: str, strings: DeviceArray, pattern, ignore_case: bool) -> DeviceArray:
    if pattern is None:
        raise pa.ArrowInvalid(f"Function '{name}' cannot be called without options")
    if not isinstance(strings, DeviceArray) or strings.type not in _BINARY_TYPES:
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({_type_name(strings)})")
    if ignore_case:
        raise pa.ArrowNotImplementedError(
            f"arrow_b200 {name}: ignore_case is not supported on the device (the reference matches with RE2's Unicode "
            "simple case folding)")
    with _string_matcher(strings.ctx, name, pattern, strings.type in _STRING_TYPES) as matcher:
        return _call(strings.ctx, "b2_string_match", pa.bool_(), C.byref(strings._c()), handle=matcher.handle)


def _string_matcher(ctx: Context, kind: str, pattern, utf8: bool) -> NativeHandle:
    raw = pattern.encode() if isinstance(pattern, str) else bytes(pattern)
    return NativeHandle(ctx, "b2_string_match_destroy", lambda h: ctx.lib.b2_string_match_create(
        ctx.handle, cabi.STRING_MATCH[kind], raw, len(raw), int(utf8), h, ctx.stream))


def match_substring(strings: DeviceArray, pattern=None, ignore_case: bool = False) -> DeviceArray:
    """match_substring: whether each string contains pattern (bytes; "" matches every string)."""
    return _string_match("match_substring", strings, pattern, ignore_case)


def starts_with(strings: DeviceArray, pattern=None, ignore_case: bool = False) -> DeviceArray:
    """starts_with: whether each string begins with pattern."""
    return _string_match("starts_with", strings, pattern, ignore_case)


def ends_with(strings: DeviceArray, pattern=None, ignore_case: bool = False) -> DeviceArray:
    """ends_with: whether each string ends with pattern."""
    return _string_match("ends_with", strings, pattern, ignore_case)


def match_like(strings: DeviceArray, pattern=None, ignore_case: bool = False) -> DeviceArray:
    """match_like: SQL LIKE (`%` any run, `_` one code point over utf8 / one byte over binary, `\\` escapes).  Over
    utf8 a pattern that is not valid UTF-8 raises ArrowInvalid, as the reference's regex compile does."""
    return _string_match("match_like", strings, pattern, ignore_case)


def string_match_plan(pattern, utf8: bool = True, kind: str = "match_like"):
    """(what the pattern runs as: "match_substring" / "starts_with" / "ends_with" / "match_like" for the general
    matcher, bytes of its literal or items of its program) as b2_string_match_create compiles it."""
    ctx, runs, nbytes = Context.get(), C.c_int32(), C.c_int64()
    with _string_matcher(ctx, kind, pattern, utf8) as matcher:
        check(ctx.lib.b2_string_match_info(matcher.handle, C.byref(runs), C.byref(nbytes)))
    names = {v: k for k, v in cabi.STRING_MATCH.items()}
    return names[runs.value], nbytes.value


# ------------------------------------------------------------------------------------
# binary_length / utf8_length / ascii_upper / ascii_lower / utf8_slice_codeunits / binary_slice /
# binary_join_element_wise (kernels/scalar_string_ascii.cc:724-880,2636-2800,3298-3420,
# kernels/scalar_string_utf8.cc:664-690,1157-1348; SliceOptions, JoinOptions compute/api_scalar.h)
# ------------------------------------------------------------------------------------
_INT64_MAX = (1 << 63) - 1


def _string_input(name: str, strings, types) -> DeviceArray:
    if not isinstance(strings, DeviceArray) or strings.type not in types:
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({_type_name(strings)})")
    return strings


def binary_length(strings: DeviceArray) -> DeviceArray:
    """binary_length: the byte length of each value, int32 (int64 for large_utf8 / large_binary)."""
    s = _string_input("binary_length", strings, _BINARY_TYPES)
    return _call(s.ctx, "b2_string_length", None, C.byref(s._c()), 0)


def utf8_length(strings: DeviceArray) -> DeviceArray:
    """utf8_length: the bytes of each value that are not UTF-8 continuation bytes (10xxxxxx), int32 or int64."""
    s = _string_input("utf8_length", strings, _STRING_TYPES)
    return _call(s.ctx, "b2_string_length", None, C.byref(s._c()), 1)


def ascii_upper(strings: DeviceArray) -> DeviceArray:
    """ascii_upper: a..z to A..Z, every other byte unchanged."""
    s = _string_input("ascii_upper", strings, _STRING_TYPES)
    return _call(s.ctx, "b2_ascii_case", s.type, C.byref(s._c()), 1)


def ascii_lower(strings: DeviceArray) -> DeviceArray:
    """ascii_lower: A..Z to a..z, every other byte unchanged."""
    s = _string_input("ascii_lower", strings, _STRING_TYPES)
    return _call(s.ctx, "b2_ascii_case", s.type, C.byref(s._c()), 0)


def _slice(name: str, strings, start, stop, step, utf8: bool) -> DeviceArray:
    if start is None:
        raise pa.ArrowInvalid(f"Function '{name}' cannot be called without options")
    s = _string_input(name, strings, _STRING_TYPES if utf8 else _BINARY_TYPES - _STRING_TYPES)
    stop = _INT64_MAX if stop is None else stop
    return _call(s.ctx, "b2_string_slice", s.type, C.byref(s._c()), int(start), int(stop), int(step), int(utf8))


def utf8_slice_codeunits(strings: DeviceArray, start=None, stop=None, step: int = 1) -> DeviceArray:
    """utf8_slice_codeunits under SliceOptions: start, stop (None: the end) and step count code points; step 0 and
    invalid UTF-8 in the part of a row the slice walks raise ArrowInvalid."""
    return _slice("utf8_slice_codeunits", strings, start, stop, step, True)


def binary_slice(strings: DeviceArray, start=None, stop=None, step: int = 1) -> DeviceArray:
    """binary_slice under SliceOptions, in bytes.  Unlike pyarrow 24, a slice with the default stop works on arrays of
    two or more rows (the reference's output estimate overflows there)."""
    return _slice("binary_slice", strings, start, stop, step, False)


def binary_join_element_wise(*strings, null_handling="emit_null", null_replacement="") -> DeviceArray:
    """binary_join_element_wise under JoinOptions: the values joined by the last argument, the separator.  Arguments are
    DeviceArrays of one type and length, or scalars (str / bytes / pa.Scalar) of that type; at least one is an array."""
    ops = [x if isinstance(x, DeviceArray) else _as_scalar(x) for x in strings]
    if not ops:
        raise pa.ArrowInvalid("VarArgs function 'binary_join_element_wise' needs at least 1 arguments but only 0 passed")
    types = [o.type for o in ops]
    if any(t != types[0] for t in types) or types[0] not in _BINARY_TYPES:
        raise pa.ArrowNotImplementedError("Function 'binary_join_element_wise' has no kernel matching input types "
                                          f"({', '.join(str(t) for t in types)})")
    arrays = [o for o in ops if isinstance(o, DeviceArray)]
    if not arrays:
        raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
    mode = _enum(null_handling, cabi.JOIN_NULL_HANDLING, "null handling behavior")
    table = (cabi.B2JoinOperand * len(ops))()
    keep = []
    for slot, o in zip(table, ops):
        if isinstance(o, DeviceArray):
            c = o._c()
            keep.append(c)
            slot.array = C.pointer(c)
        else:
            raw = o.as_buffer().to_pybytes() if o.is_valid else b""
            keep.append(raw)
            slot.bytes, slot.length, slot.is_valid = raw, len(raw), int(o.is_valid)
    repl = null_replacement.encode() if isinstance(null_replacement, str) else bytes(null_replacement)
    return _call(arrays[0].ctx, "b2_binary_join_element_wise", types[0], table, len(ops), mode, repl, len(repl))


# ------------------------------------------------------------------------------------
# calendar and clock fields (kernels/scalar_temporal_unary.cc:222-691; DayOfWeekOptions compute/api_scalar.h)
# ------------------------------------------------------------------------------------
def _zone_offset(tz: str) -> int:
    """The offset in minutes of a zone the device takes: "UTC", or a fixed offset in a form LocateZone accepts
    (kernels/temporal_internal.cc:22-45): a sign and HH:MM or HHMM, hours below 24 and minutes below 60."""
    if tz == "UTC":
        return 0
    if tz[:1] in ("+", "-"):
        body = tz[1:]
        hh, mm = body[:2], body[-2:]
        if (len(body) not in (4, 5) or (len(body) == 5 and body[2] != ":") or not (hh + mm).isdecimal() or int(hh) > 23
                or int(mm) > 59):
            raise pa.ArrowInvalid(f"Cannot locate or parse timezone '{tz}'")
        minutes = int(hh) * 60 + int(mm)
        return -minutes if tz[0] == "-" else minutes
    raise pa.ArrowNotImplementedError(
        f"arrow_b200: time zone '{tz}' is not supported on the device (only UTC and fixed offsets such as +05:30)")


def temporal_type(t: pa.DataType) -> "cabi.B2TemporalType":
    """The B2TemporalType descriptor of a temporal (or int32 / int64) type; a named zone raises NotImplemented."""
    d = cabi.B2TemporalType(0, 0, 0, 0)
    if pa.types.is_date32(t) or pa.types.is_date64(t) or t in (pa.int32(), pa.int64()):
        d.kind = cabi.TEMPORAL_KINDS[str(t).split("[")[0]]
        return d
    for kind, pred in (("time32", pa.types.is_time32), ("time64", pa.types.is_time64),
                       ("timestamp", pa.types.is_timestamp), ("duration", pa.types.is_duration)):
        if pred(t):
            d.kind, d.unit = cabi.TEMPORAL_KINDS[kind], cabi.TIME_UNITS[t.unit]
            if kind == "timestamp" and t.tz is not None:
                d.has_zone, d.offset_minutes = 1, _zone_offset(t.tz)
            return d
    raise pa.ArrowNotImplementedError(f"arrow_b200: {t} is not a temporal type")


def _temporal_field(name: str, arr: DeviceArray, week_start: int = 1, count_from_zero: bool = True) -> DeviceArray:
    if not isinstance(arr, DeviceArray):
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({_type_name(arr)})")
    try:
        desc = temporal_type(arr.type)
    except pa.ArrowNotImplementedError:
        if pa.types.is_timestamp(arr.type):
            raise
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({arr.type})") from None
    if desc.kind in (cabi.TEMPORAL_KINDS["int32"], cabi.TEMPORAL_KINDS["int64"]):
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({arr.type})")
    out_type = pa.bool_() if name == "is_leap_year" else pa.float64() if name == "subsecond" else pa.int64()
    return _call(arr.ctx, "b2_temporal_field", out_type, C.byref(arr._c()), C.byref(desc), cabi.TEMPORAL_FIELDS[name],
                 int(week_start), int(bool(count_from_zero)))


def year(arr): return _temporal_field("year", arr)
def month(arr): return _temporal_field("month", arr)
def day(arr): return _temporal_field("day", arr)
def day_of_year(arr): return _temporal_field("day_of_year", arr)
def quarter(arr): return _temporal_field("quarter", arr)
def is_leap_year(arr): return _temporal_field("is_leap_year", arr)
def hour(arr): return _temporal_field("hour", arr)
def minute(arr): return _temporal_field("minute", arr)
def second(arr): return _temporal_field("second", arr)
def millisecond(arr): return _temporal_field("millisecond", arr)
def microsecond(arr): return _temporal_field("microsecond", arr)
def nanosecond(arr): return _temporal_field("nanosecond", arr)
def subsecond(arr): return _temporal_field("subsecond", arr)


def day_of_week(arr, count_from_zero: bool = True, week_start: int = 1):
    """day_of_week under DayOfWeekOptions: Monday = 0 (or 1 without count_from_zero) when week_start is 1 (Monday);
    week_start outside 1..7 raises ArrowInvalid."""
    return _temporal_field("day_of_week", arr, week_start, count_from_zero)


# ------------------------------------------------------------------------------------
# numeric math (kernels/base_arithmetic_internal.h, kernels/scalar_arithmetic.cc, kernels/scalar_round.cc)
# ------------------------------------------------------------------------------------
_FLOAT_IDS = (cabi.FLOAT, cabi.DOUBLE)
_TO_FLOAT = ("sqrt", "sqrt_checked", "floor", "ceil", "trunc")


def _math_input(name: str, x) -> DeviceArray:
    if not isinstance(x, DeviceArray):
        raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
    if x.type not in _NUMERIC_TYPES:
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({x.type})")
    return x


def _unary(name: str, x) -> DeviceArray:
    x = _math_input(name, x)
    tid = type_id(x.type)
    if name in _TO_FLOAT and tid not in _FLOAT_IDS:  # an integer is cast to float64 first (DispatchBest)
        x, tid = cast(x, pa.float64()), cabi.DOUBLE
    out_type = pa.int8() if name == "sign" and tid not in _FLOAT_IDS else x.type
    return _call(x.ctx, "b2_unary_arith", out_type, cabi.UNARY_OPS[name], C.byref(x._c()))


def abs(x): return _unary("abs", x)  # noqa: A001
def abs_checked(x): return _unary("abs_checked", x)
def negate(x): return _unary("negate", x)
def negate_checked(x): return _unary("negate_checked", x)
def sign(x): return _unary("sign", x)
def sqrt(x): return _unary("sqrt", x)
def sqrt_checked(x): return _unary("sqrt_checked", x)
def floor(x): return _unary("floor", x)
def ceil(x): return _unary("ceil", x)
def trunc(x): return _unary("trunc", x)
def bit_wise_not(x): return _unary("bit_wise_not", x)


def _integer_arith(name: str, x, y) -> DeviceArray:
    """power, the bit-wise ops and the shifts: integers only, over the operands' common numeric type.  Float power is
    not on the device (its libm and CUDA results may differ in the last bits)."""
    _, tid = _numeric_operands(x, y)
    if tid in _FLOAT_IDS:
        raise pa.ArrowNotImplementedError(
            f"Function '{name}' has no kernel matching input types ({_type_name(x)}, {_type_name(y)})")
    return _arith(name, x, y)


def power(base, exponent): return _integer_arith("power", base, exponent)
def power_checked(base, exponent): return _integer_arith("power_checked", base, exponent)
def bit_wise_and(x, y): return _integer_arith("bit_wise_and", x, y)
def bit_wise_or(x, y): return _integer_arith("bit_wise_or", x, y)
def bit_wise_xor(x, y): return _integer_arith("bit_wise_xor", x, y)
def shift_left(x, y): return _integer_arith("shift_left", x, y)
def shift_left_checked(x, y): return _integer_arith("shift_left_checked", x, y)
def shift_right(x, y): return _integer_arith("shift_right", x, y)
def shift_right_checked(x, y): return _integer_arith("shift_right_checked", x, y)


def _round_mode(round_mode) -> int:
    return _enum(round_mode, cabi.ROUND_MODES, "round mode")


def round(x, ndigits: int = 0, round_mode="half_to_even") -> DeviceArray:  # noqa: A001
    """round under RoundOptions: a float is scaled by 10^ndigits, rounded in round_mode and scaled back, by the
    reference's operations (so round(0.7, 11) is 0.699999999996, as in pyarrow 24); an integer stays one, rounded to a
    multiple of 10^-ndigits when ndigits < 0."""
    x = _math_input("round", x)
    keep = []
    return _call(x.ctx, "b2_round", x.type, C.byref(_value(x, type_id(x.type), keep)), None, int(ndigits), None,
                 _round_mode(round_mode))


def round_to_multiple(x, multiple=1.0, round_mode="half_to_even") -> DeviceArray:
    """round_to_multiple under RoundToMultipleOptions: the multiple must be valid and positive, and is cast safely to
    x's type."""
    x = _math_input("round_to_multiple", x)
    m = _as_scalar(multiple)
    if not m.is_valid:
        raise pa.ArrowInvalid("Rounding multiple must be non-null and valid")
    if m.type not in _NUMERIC_TYPES or not m.as_py() > 0:
        raise pa.ArrowInvalid("Rounding multiple must be positive")
    sm = _scalar_to(m, type_id(x.type))
    keep = []
    return _call(x.ctx, "b2_round", x.type, C.byref(_value(x, type_id(x.type), keep)), None, 0, C.byref(sm),
                 _round_mode(round_mode))


def round_binary(x, s, round_mode="half_to_even") -> DeviceArray:
    """round_binary under RoundBinaryOptions: round(x, s) with the digit count s per row, cast to int32.  A float is
    scaled in float64 whatever its type."""
    xo = x if isinstance(x, DeviceArray) else _as_scalar(x)
    so = s if isinstance(s, DeviceArray) else _as_scalar(s)
    if pa.types.is_null(so.type):
        so = pa.scalar(None, pa.int32())
    if xo.type not in _NUMERIC_TYPES or so.type not in _NUMERIC_TYPES:
        raise pa.ArrowNotImplementedError(
            f"Function 'round_binary' has no kernel matching input types ({xo.type}, {so.type})")
    if not isinstance(xo, DeviceArray) and not isinstance(so, DeviceArray):
        raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
    keep = []
    tid = type_id(xo.type)
    vx, vs = _value(xo, tid, keep), _value(so, cabi.INT32, keep)
    ctx = xo.ctx if isinstance(xo, DeviceArray) else so.ctx
    return _call(ctx, "b2_round", xo.type, C.byref(vx), C.byref(vs), 0, None, _round_mode(round_mode))


# ------------------------------------------------------------------------------------
# cumulative functions (kernels/vector_cumulative_ops.cc; CumulativeOptions compute/api_vector.h:335-355)
# ------------------------------------------------------------------------------------
def _cumulative(name: str, values, start, skip_nulls: bool) -> DeviceArray:
    """One output over a DeviceArray or the list of chunks of one column, the state carried from chunk to chunk as
    CumulativeKernelChunked does.  `start` is cast to the values' type by pyarrow's safe cast (CumulativeOptionsWrapper
    ::Init), so its errors are the reference's; cumulative_mean ignores it."""
    chunks = [values] if isinstance(values, DeviceArray) else list(values)
    if not chunks or not builtins.all(isinstance(c, DeviceArray) for c in chunks):
        raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: values must be a device array or a non-empty list of them")
    t = chunks[0].type
    if t not in _NUMERIC_TYPES or builtins.any(c.type != t for c in chunks):
        raise pa.ArrowNotImplementedError(f"Function '{name}' has no kernel matching input types ({t})")
    cstart = None
    if start is not None:  # cast for cumulative_mean too, as the reference does, though the mean ignores it
        cstart = _scalar_to(_as_scalar(start).cast(t, safe=True), type_id(t))
        if name == "cumulative_mean":
            cstart = None
    ctx = chunks[0].ctx
    carr = (cabi.B2Array * len(chunks))(*[c._c() for c in chunks])
    out_type = pa.float64() if name == "cumulative_mean" else t
    return _call(ctx, "b2_cumulative", out_type, cabi.CUMULATIVE_OPS[name], carr, len(chunks),
                 None if cstart is None else C.byref(cstart), 1 if skip_nulls else 0)


def cumulative_sum(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_sum", values, start, skip_nulls)


def cumulative_sum_checked(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_sum_checked", values, start, skip_nulls)


def cumulative_prod(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_prod", values, start, skip_nulls)


def cumulative_prod_checked(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_prod_checked", values, start, skip_nulls)


def cumulative_min(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_min", values, start, skip_nulls)


def cumulative_max(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_max", values, start, skip_nulls)


def cumulative_mean(values, start=None, skip_nulls: bool = False):
    return _cumulative("cumulative_mean", values, start, skip_nulls)


# ------------------------------------------------------------------------------------
# grouper + hash aggregates
# ------------------------------------------------------------------------------------
class Grouper(NativeHandle):
    """arrow::compute::Grouper (compute/row/grouper.h:104-196) over fixed-width and utf8 / binary key columns."""

    def __init__(self, key_types: Sequence[pa.DataType], ctx: Optional[Context] = None):
        ctx = ctx or Context.get()
        self.key_types = [pa.lib.ensure_type(t) for t in key_types]
        ids = (C.c_int32 * len(self.key_types))(*[type_id(t) for t in self.key_types])
        super().__init__(ctx, "b2_grouper_destroy", lambda h: ctx.lib.b2_grouper_create(ctx.handle, ids, len(ids), h))

    def _keys(self, keys):
        if isinstance(keys, DeviceArray):
            keys = [keys]
        if len(keys) != len(self.key_types):
            raise pa.ArrowInvalid(f"expected batch size {len(self.key_types)} but got {len(keys)}")
        for k, t in zip(keys, self.key_types):
            if k.type != t:
                raise pa.ArrowInvalid(f"expected batch value of type {t} but got {k.type}")
        return (cabi.B2Array * len(keys))(*[k._c() for k in keys])

    def consume(self, keys) -> DeviceArray:
        return _call(self.ctx, "b2_grouper_consume", pa.uint32(), self._keys(keys), handle=self.handle)

    def lookup(self, keys) -> DeviceArray:
        return _call(self.ctx, "b2_grouper_lookup", pa.uint32(), self._keys(keys), handle=self.handle)

    @property
    def num_groups(self) -> int:
        n = C.c_uint32()
        check(self.ctx.lib.b2_grouper_num_groups(self.handle, C.byref(n)))
        return n.value

    def get_uniques(self):
        couts = (cabi.B2Array * len(self.key_types))()
        check(self.ctx.lib.b2_grouper_uniques(self.handle, couts, self.ctx.stream))
        return [_out(self.ctx, couts[i], t) for i, t in enumerate(self.key_types)]

    def reset(self):
        check(self.ctx.lib.b2_grouper_reset(self.handle))

    @staticmethod
    def make_groupings(ids: DeviceArray, num_groups: int) -> DeviceArray:
        """Grouper::MakeGroupings (compute/row/grouper.h:141-167): list<int32> of length num_groups whose entry g holds
        the row numbers with id g, in row order.  Null ids raise ArrowInvalid, an id >= num_groups ArrowIndexError, more
        than 2^31 - 1 ids ArrowCapacityError."""
        ctx = ids.ctx
        ci, co, cr = ids._c(), cabi.B2Array(), cabi.B2Array()
        check(ctx.lib.b2_make_groupings(ctx.handle, C.byref(ci), int(num_groups), C.byref(co), C.byref(cr), ctx.stream))
        return _list(ctx, co, _out(ctx, cr, pa.int32()), pa.int32())

    @staticmethod
    def apply_groupings(groupings: DeviceArray, values: DeviceArray) -> DeviceArray:
        """Grouper::ApplyGroupings (grouper.h:169-194): values gathered through the groupings' rows, as a list<values.type>
        under the groupings' offsets.  The rows are bounds-checked: they may come from outside this module."""
        if not pa.types.is_list(groupings.type) or groupings.type.value_type != pa.int32():
            raise pa.ArrowTypeError(f"groupings must be list<int32>, got {groupings.type}")
        child = take(values, groupings.children[0])
        return DeviceArray(values.ctx, pa.list_(values.type), groupings.length, 0, groupings.offset,
                           [None, groupings.buffers[1]], children=[child])


JOIN_TYPES = {"inner": 0, "left outer": 1, "left semi": 2, "left anti": 3, "full outer": 4}


def hash_join_indices(left_keys: Sequence[DeviceArray], right_keys: Sequence[DeviceArray], join_type: str = "inner",
                      key_cmp: Optional[Sequence[str]] = None, residual=None):
    """The matching row pairs of an equi-join (the build / probe / match core of acero's HashJoinNode, hash_join_node.cc;
    join types as pyarrow.Table.join spells them).  Returns (left_indices, right_indices) as uint32 DeviceArrays -- for
    "left outer" right_indices is null where a left row found no match ("full outer" appends the unmatched right rows with a
    null left index), for "left semi" / "left anti" right_indices is None.
    key_cmp: None (every column "eq"), or one "eq" / "is" per key column (JoinKeyCmp): with "eq" a null key matches nothing,
    with "is" a null equals a null.
    residual: None, or a callable (left_rows, right_rows) -> boolean DeviceArray, one flag per candidate pair (HashJoinNodeOptions
    filter): it gets the uint32 rows of every key-matching pair, gathers what it needs with take() and evaluates the predicate
    on the device.  A pair survives only where the flag is true (null counts as false); a left row whose pairs all fail is
    unmatched.  Gather the payload columns with take()."""
    if isinstance(left_keys, DeviceArray):
        left_keys = [left_keys]
    if isinstance(right_keys, DeviceArray):
        right_keys = [right_keys]
    if join_type not in JOIN_TYPES:
        raise ValueError(f'"{join_type}" is not a supported join type ({", ".join(JOIN_TYPES)})')
    if len(left_keys) != len(right_keys) or not left_keys:
        raise pa.ArrowInvalid("join needs the same, non-zero number of key columns on both sides")
    for l, r in zip(left_keys, right_keys):
        if l.type != r.type:
            raise pa.ArrowInvalid(f"Incompatible data types for corresponding join field keys: {l.type} and {r.type}")
    null_equal = None
    if key_cmp is not None:
        key_cmp = list(key_cmp)
        if len(key_cmp) != len(left_keys) or any(c not in ("eq", "is") for c in key_cmp):
            raise ValueError(f'key_cmp needs one "eq" or "is" per key column, got {key_cmp}')
        if "is" in key_cmp:
            null_equal = (C.c_uint8 * len(key_cmp))(*[int(c == "is") for c in key_cmp])
    ctx = left_keys[0].ctx
    cl = (cabi.B2Array * len(left_keys))(*[k._c() for k in left_keys])
    cr = (cabi.B2Array * len(right_keys))(*[k._c() for k in right_keys])
    ol, orr = cabi.B2Array(), cabi.B2Array()
    jt = JOIN_TYPES[join_type]
    pairs = jt in (0, 1, 4)
    if residual is None and null_equal is None:
        check(ctx.lib.b2_hash_join(ctx.handle, cl, cr, len(left_keys), jt, C.byref(ol), C.byref(orr) if pairs else None, ctx.stream))
        return _out(ctx, ol, pa.uint32()), (_out(ctx, orr, pa.uint32()) if pairs else None)
    if residual is None:
        check(ctx.lib.b2_hash_join_ex(ctx.handle, cl, cr, len(left_keys), null_equal, jt, C.byref(ol), C.byref(orr) if pairs else None,
                                      ctx.stream))
        return _out(ctx, ol, pa.uint32()), (_out(ctx, orr, pa.uint32()) if pairs else None)
    check(ctx.lib.b2_hash_join_ex(ctx.handle, cl, cr, len(left_keys), null_equal, 0, C.byref(ol), C.byref(orr), ctx.stream))
    cand_l, cand_r = _out(ctx, ol, pa.uint32()), _out(ctx, orr, pa.uint32())
    keep = residual(cand_l, cand_r)
    if not isinstance(keep, DeviceArray) or not pa.types.is_boolean(keep.type):
        raise pa.ArrowTypeError(f"the residual filter must return a boolean DeviceArray, got {getattr(keep, 'type', type(keep))}")
    return join_residual(cand_l, cand_r, keep, len(left_keys[0]), len(right_keys[0]), join_type)


def join_residual(cand_left: DeviceArray, cand_right: DeviceArray, keep: DeviceArray, n_left: int, n_right: int,
                  join_type: str = "inner"):
    """The join_type result over the candidate pairs whose keep flag is true (b2_join_residual): cand_left / cand_right are
    the "inner" pairs of hash_join_indices (uint32, left rows non-decreasing), n_left / n_right the side lengths.  Same
    order and layout as hash_join_indices; invalid pairs raise ArrowInvalid before anything is written."""
    if join_type not in JOIN_TYPES:
        raise ValueError(f'"{join_type}" is not a supported join type ({", ".join(JOIN_TYPES)})')
    ctx = cand_left.ctx
    jt = JOIN_TYPES[join_type]
    pairs = jt in (0, 1, 4)
    a, b, k = cand_left._c(), cand_right._c(), keep._c()
    ol, orr = cabi.B2Array(), cabi.B2Array()
    check(ctx.lib.b2_join_residual(ctx.handle, C.byref(a), C.byref(b), C.byref(k), int(n_left), int(n_right), jt, C.byref(ol),
                                   C.byref(orr) if pairs else None, ctx.stream))
    return _out(ctx, ol, pa.uint32()), (_out(ctx, orr, pa.uint32()) if pairs else None)


_MOMENT_FUNCTIONS = ("hash_variance", "hash_stddev", "hash_skew", "hash_kurtosis")


class HashAggregator(NativeHandle):
    """One HashAggregateKernel state (compute/kernel.h:720-769): resize/consume/merge/finalize.

    hash_variance / hash_stddev take ddof=, hash_skew / hash_kurtosis take biased=; for these four min_count defaults
    to 0 (VarianceOptions / SkewOptions, api_aggregate.h:103-134), for the others to 1.  hash_list and hash_distinct
    (mode= as hash_count_distinct) finalize to a list<value_type>."""

    def __init__(self, function: str, value_type: Optional[pa.DataType], *, skip_nulls=True, min_count=None,
                 mode="only_valid", ddof=0, biased=True, ctx: Optional[Context] = None):
        ctx = ctx or Context.get()
        self.function = function
        self.value_type = value_type
        kind = cabi.HASH_AGG_KINDS[function]
        cm = _COUNT_MODE[mode]
        moments = function in _MOMENT_FUNCTIONS
        if min_count is None:
            min_count = 0 if moments else 1
        if function in ("hash_variance", "hash_stddev"):
            if int(ddof) < 0:
                raise pa.ArrowInvalid(f"ddof must be >= 0, got {ddof}")
            param = int(ddof)
        elif function in ("hash_skew", "hash_kurtosis"):
            param = 0 if biased else 1
        else:
            param = 0
        opts = cabi.B2HashAggOptions(int(skip_nulls), int(min_count), cm, param)
        vt = type_id(value_type) if value_type is not None else cabi.NA
        super().__init__(ctx, "b2_hashagg_destroy", lambda h: ctx.lib.b2_hashagg_create(ctx.handle, kind, vt, C.byref(opts), h))

    def resize(self, num_groups: int):
        check(self.ctx.lib.b2_hashagg_resize(self.handle, int(num_groups), self.ctx.stream))

    def consume(self, values: Optional[DeviceArray], ids: Optional[DeviceArray]):
        """ids=None: every row is in group 0 (the moment functions over a state of one group)"""
        cv = values._c() if values is not None else None
        ci = ids._c() if ids is not None else None
        check(self.ctx.lib.b2_hashagg_consume(self.handle, C.byref(cv) if cv is not None else None,
                                              C.byref(ci) if ci is not None else None, self.ctx.stream))

    def merge(self, other: "HashAggregator", group_id_mapping: DeviceArray):
        cm = group_id_mapping._c()
        check(self.ctx.lib.b2_hashagg_merge(self.handle, other.handle, C.byref(cm), self.ctx.stream))

    def finalize(self) -> DeviceArray:
        if self.function in ("hash_list", "hash_distinct"):
            co, cv = cabi.B2Array(), cabi.B2Array()
            check(self.ctx.lib.b2_hashagg_finalize_list(self.handle, C.byref(co), C.byref(cv), self.ctx.stream))
            return _list(self.ctx, co, _out(self.ctx, cv, self.value_type), self.value_type)
        return _call(self.ctx, "b2_hashagg_finalize", None, handle=self.handle)


def group_by(keys: Sequence[DeviceArray], aggregates: Sequence[tuple], fused: bool = True):
    """The Acero aggregate node's Consume/Finalize over one batch
    (acero/groupby_aggregate_node.cc:210-253,300-337): aggregates = [(function, values|None, opts)].
    Returns (unique key columns, [aggregate columns]); group order is unspecified (as under use_threads in the
    reference, whose tests sort by key)."""
    if isinstance(keys, DeviceArray):
        keys = [keys]
    # config 3's shape -- one fixed-width key, hash_sum / hash_count(only_valid) / hash_mean with default options over
    # one value column -- takes the fused path (b2_groupby_sumcount_*), exactly as the C++ b200_aggregate node does;
    # pass fused=False or any option to force the Grouper path.  hash_mean = sum / count of the same state; 64-bit
    # integer columns keep the unfused kernel (the reference's mean accumulates in double,
    # hash_aggregate_numeric.cc:353-356, which an exact int64 sum that wraps would not match).
    if fused and len(keys) == 1 and aggregates and all(
            fn in ("hash_sum", "hash_count", "hash_mean") and values is not None and not opts and values is aggregates[0][1]
            for fn, values, opts in aggregates) and keys[0].type in _NUMERIC_TYPES and aggregates[0][1].type in _NUMERIC_TYPES \
            and not pa.types.is_floating(keys[0].type) \
            and not (any(fn == "hash_mean" for fn, _, _ in aggregates) and aggregates[0][1].type in (pa.int64(), pa.uint64())):
        gb = GroupBySumCount(keys[0].type, aggregates[0][1].type, ctx=keys[0].ctx)
        gb.consume(keys[0], aggregates[0][1])
        k, s_, c_ = gb.finalize()
        m_ = None
        if any(fn == "hash_mean" for fn, _, _ in aggregates):
            m_ = divide(cast(s_, pa.float64(), safe=False), cast(c_, pa.float64(), safe=False))
        return [k], [{"hash_sum": s_, "hash_count": c_, "hash_mean": m_}[fn] for fn, _, _ in aggregates]
    g = Grouper([k.type for k in keys], keys[0].ctx)
    ids = g.consume(keys)
    outs = []
    for fn, values, opts in aggregates:
        agg = HashAggregator(fn, values.type if values is not None else None, ctx=keys[0].ctx, **(opts or {}))
        agg.resize(g.num_groups)
        agg.consume(values, ids)
        outs.append(agg.finalize())
    return g.get_uniques(), outs


def _moment_scalar(function: str, arrays, **opts) -> pa.Scalar:
    """The ungrouped statistic: a one-group aggregator fed without ids, one consume per chunk."""
    if isinstance(arrays, DeviceArray):
        arrays = [arrays]
    for a in arrays:
        _require_numeric(a.type)
    agg = HashAggregator("hash_" + function, arrays[0].type, ctx=arrays[0].ctx, **opts)
    agg.resize(1)
    for a in arrays:
        agg.consume(a, None)
    return agg.finalize().to_arrow()[0]


def variance(arr: DeviceArray, ddof: int = 0, skip_nulls: bool = True, min_count: int = 0) -> pa.Scalar:
    """variance (VarianceImpl, kernels/aggregate_var_std.cc:40-235; VarianceOptions api_aggregate.h:103-117) as float64.
    A list of chunks is consumed batch by batch, as the reference consumes a ChunkedArray."""
    return _moment_scalar("variance", arr, ddof=ddof, skip_nulls=skip_nulls, min_count=min_count)


def stddev(arr: DeviceArray, ddof: int = 0, skip_nulls: bool = True, min_count: int = 0) -> pa.Scalar:
    """stddev: sqrt(variance) (aggregate_var_std.cc:40-235)."""
    return _moment_scalar("stddev", arr, ddof=ddof, skip_nulls=skip_nulls, min_count=min_count)


def skew(arr: DeviceArray, skip_nulls: bool = True, biased: bool = True, min_count: int = 0) -> pa.Scalar:
    """skew (aggregate_var_std.cc:40-235; SkewOptions api_aggregate.h:119-134)."""
    return _moment_scalar("skew", arr, skip_nulls=skip_nulls, biased=biased, min_count=min_count)


def kurtosis(arr: DeviceArray, skip_nulls: bool = True, biased: bool = True, min_count: int = 0) -> pa.Scalar:
    """kurtosis, excess (aggregate_var_std.cc:40-235; SkewOptions api_aggregate.h:119-134)."""
    return _moment_scalar("kurtosis", arr, skip_nulls=skip_nulls, biased=biased, min_count=min_count)


class GroupBySumCount(NativeHandle):
    """Fused consume of the aggregate node for `hash_sum` + `hash_count` over one value column
    (b2_groupby_sumcount_*): same results as Grouper + two HashAggregators."""

    def __init__(self, key_type, value_type, expected_groups=0, ctx: Optional[Context] = None):
        ctx = ctx or Context.get()
        self.key_type, self.value_type = pa.lib.ensure_type(key_type), pa.lib.ensure_type(value_type)
        kt, vt = type_id(self.key_type), type_id(self.value_type)
        super().__init__(ctx, "b2_groupby_sumcount_destroy",
                         lambda h: ctx.lib.b2_groupby_sumcount_create(ctx.handle, kt, vt, int(expected_groups), h))

    def consume(self, keys: DeviceArray, values: DeviceArray):
        ck, cv = keys._c(), values._c()
        check(self.ctx.lib.b2_groupby_sumcount_consume(self.handle, C.byref(ck), C.byref(cv), self.ctx.stream))

    def merge(self, keys: DeviceArray, sums: DeviceArray, counts: DeviceArray):
        """add partial (key, sum, count) states of another group-by (HashAggregateKernel::merge for the fused table)"""
        ck, cs, cc = keys._c(), sums._c(), counts._c()
        check(self.ctx.lib.b2_groupby_sumcount_merge(self.handle, C.byref(ck), C.byref(cs), C.byref(cc), self.ctx.stream))

    def path_counts(self):
        """{dense, compact, general, atomic}: chunks consumed so far by each internal path"""
        d, a, b, c = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        check(self.ctx.lib.b2_groupby_sumcount_path_counts(self.handle, C.byref(d), C.byref(a), C.byref(b), C.byref(c)))
        return {"dense": d.value, "compact": a.value, "general": b.value, "atomic": c.value}

    def finalize(self):
        k, s, c = cabi.B2Array(), cabi.B2Array(), cabi.B2Array()
        check(self.ctx.lib.b2_groupby_sumcount_finalize(self.handle, C.byref(k), C.byref(s), C.byref(c),
                                                        self.ctx.stream))
        return (_out(self.ctx, k, self.key_type), _out(self.ctx, s, arrow_type(s.type)),
                _out(self.ctx, c, pa.int64()))


# ------------------------------------------------------------------------------------
# CallFunction-style registry (compute/registry.cc:87-96 lookup by name)
# ------------------------------------------------------------------------------------
def _read_options(name: str, options, cls: str, fields: dict) -> dict:
    """A function's options as its keywords.  A dict holds the keywords themselves.  pyarrow's Options classes expose no
    attributes, so a `cls` object is read from its repr ('MatchSubstringOptions(pattern="ab", ignore_case=false)'):
    `fields` maps each field of that repr, in its order, to the keyword it is passed as (None: not passed)."""
    if isinstance(options, dict):
        return dict(options)
    m = re.fullmatch(cls + r"\(" + ", ".join(f + "=(.*)" for f in fields) + r"\)", str(options), re.S)
    if m is None:
        raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: pass the {cls} fields as a dict")
    out = {}
    for keyword, text in zip(fields.values(), m.groups()):
        if text in ("true", "false"):
            value = text == "true"
        elif re.fullmatch(r"-?\d+", text):
            value = int(text)
        elif text[:1] == '"':
            value = text[1:-1]
        elif text[:1] == "[":  # sort keys: [FieldRef.Name(x) DESC, ...]
            value = [(key, "descending" if o == "DESC" else "ascending")
                     for key, o in re.findall(r"FieldRef\.Name\((.*?)\) (ASC|DESC)", text)]
        else:  # an enum (EMIT_NULL, AtStart) or type name, as the Python API spells it; CountOptions spells two modes apart
            value = re.sub(r"(?<=[a-z])(?=[A-Z])", "_", text).lower()
            value = {"non_null": "only_valid", "nulls": "only_null"}.get(value, value)
        if keyword is not None:
            out[keyword] = value
    return out


def _options(cls: str, *fields: str):
    """The options adapter of a function whose keywords are the fields of pyarrow's `cls`, in the order of its repr."""
    return lambda name, options: _read_options(name, options, cls, {f: f for f in fields})


def _cast_options(name: str, options) -> dict:
    """CastOptions exposes its flags but not its target type, which is read from the repr."""
    if isinstance(options, dict):
        return dict(options)
    fields = dict.fromkeys(("to_type", "allow_int_overflow", "allow_time_truncate", "allow_time_overflow",
                            "allow_decimal_truncate", "allow_float_truncate", "allow_invalid_utf8"))
    fields["to_type"] = "target_type"
    return {**_read_options(name, options, "CastOptions", fields), "options": options}


def _set_lookup_options(name: str, options) -> dict:
    # pyarrow's SetLookupOptions exposes no attributes and its repr cannot carry the value set: a dict is required
    if not isinstance(options, dict):
        raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: pass the SetLookupOptions fields as a dict "
                                          "(value_set, skip_nulls, null_matching_behavior)")
    return options


_FILTER = _options("FilterOptions", "null_selection_behavior")
_TAKE = _options("TakeOptions", "boundscheck")
_SCALAR_AGGREGATE = _options("ScalarAggregateOptions", "skip_nulls", "min_count")
_VARIANCE = _options("VarianceOptions", "ddof", "skip_nulls", "min_count")
_SKEW = _options("SkewOptions", "skip_nulls", "biased", "min_count")
_COUNT = _options("CountOptions", "mode")
_MATCH = _options("MatchSubstringOptions", "pattern", "ignore_case")
_SLICE = _options("SliceOptions", "start", "stop", "step")

# name: (function, adapter from its options to its keywords, None for a function without options)
_REGISTRY = {
    "cast": (cast, _cast_options), "filter": (filter, _FILTER), "array_filter": (array_filter, _FILTER),
    "take": (take, _TAKE), "array_take": (array_take, _TAKE),
    "sort_indices": (sort_indices, _options("SortOptions", "sort_keys", "null_placement")),
    "array_sort_indices": (array_sort_indices, _options("ArraySortOptions", "order", "null_placement")),
    "select_k_unstable": (select_k_unstable, _options("SelectKOptions", "k", "sort_keys")),
    "if_else": (if_else, None),
    "add": (add, None), "subtract": (subtract, None), "multiply": (multiply, None), "divide": (divide, None),
    "add_checked": (add_checked, None), "subtract_checked": (subtract_checked, None),
    "multiply_checked": (multiply_checked, None), "divide_checked": (divide_checked, None),
    "equal": (equal, None), "not_equal": (not_equal, None), "greater": (greater, None),
    "greater_equal": (greater_equal, None), "less": (less, None), "less_equal": (less_equal, None),
    "unique": (unique, None), "value_counts": (value_counts, None),
    "dictionary_encode": (dictionary_encode, lambda name, options: _read_options(
        name, options, "DictionaryEncodeOptions", {"null_encoding_behavior": "null_encoding"})),
    "count_distinct": (count_distinct, _COUNT),
    "is_in": (is_in, _set_lookup_options), "index_in": (index_in, _set_lookup_options),
    "match_substring": (match_substring, _MATCH), "starts_with": (starts_with, _MATCH), "ends_with": (ends_with, _MATCH),
    "match_like": (match_like, _MATCH),
    "binary_length": (binary_length, None), "utf8_length": (utf8_length, None), "ascii_upper": (ascii_upper, None),
    "ascii_lower": (ascii_lower, None),
    "year": (year, None), "month": (month, None), "day": (day, None), "day_of_year": (day_of_year, None),
    "day_of_week": (day_of_week, _options("DayOfWeekOptions", "count_from_zero", "week_start")),
    "quarter": (quarter, None), "is_leap_year": (is_leap_year, None), "hour": (hour, None), "minute": (minute, None),
    "second": (second, None), "millisecond": (millisecond, None), "microsecond": (microsecond, None),
    "nanosecond": (nanosecond, None), "subsecond": (subsecond, None),
    "sum": (sum, _SCALAR_AGGREGATE), "mean": (mean, _SCALAR_AGGREGATE), "min_max": (min_max, _SCALAR_AGGREGATE),
    "min": (min, _SCALAR_AGGREGATE), "max": (max, _SCALAR_AGGREGATE), "count": (count, _COUNT),
    "variance": (variance, _VARIANCE), "stddev": (stddev, _VARIANCE), "skew": (skew, _SKEW), "kurtosis": (kurtosis, _SKEW),
    "and": (and_, None), "or": (or_, None), "xor": (xor, None), "and_not": (and_not, None),
    "and_kleene": (and_kleene, None), "or_kleene": (or_kleene, None), "and_not_kleene": (and_not_kleene, None),
    "invert": (invert, None), "is_valid": (is_valid, None), "is_null": (is_null, _options("NullOptions", "nan_is_null")),
    "true_unless_null": (true_unless_null, None), "is_nan": (is_nan, None),
}


# The string transforms that take options.  tests/test_cabi_enums.py checks the option-taking entries of _REGISTRY
# against a fixed list of cases, and tests/test_gpu_string_transform.py checks these three the same way; call_function
# and list_functions see one table, _FUNCTIONS.
_STRING_TRANSFORM_OPTIONS = {
    "utf8_slice_codeunits": (utf8_slice_codeunits, _SLICE), "binary_slice": (binary_slice, _SLICE),
    "binary_join_element_wise": (binary_join_element_wise, _options("JoinOptions", "null_handling", "null_replacement")),
}


def _round_to_multiple_options(name: str, options) -> dict:
    """RoundToMultipleOptions' repr writes the multiple as 'type:value' ('int64:10', 'double:0.5')."""
    out = _read_options(name, options, "RoundToMultipleOptions", {"multiple": "multiple", "round_mode": "round_mode"})
    if not isinstance(options, dict):
        tname, _, text = str(out["multiple"]).partition(":")
        t = pa.type_for_alias(tname)
        out["multiple"] = pa.scalar(None if text == "null" else (float(text) if pa.types.is_floating(t) else int(text)), t)
    return out


# The numeric math functions: those that take options sit apart from _REGISTRY for the reason given above, and
# tests/test_gpu_math.py checks their options forms.
_MATH_FUNCTIONS = {
    name: (globals()[name], None) for name in (
        "abs", "abs_checked", "negate", "negate_checked", "sign", "sqrt", "sqrt_checked", "floor", "ceil", "trunc",
        "bit_wise_not", "power", "power_checked", "bit_wise_and", "bit_wise_or", "bit_wise_xor", "shift_left",
        "shift_left_checked", "shift_right", "shift_right_checked")
}
_MATH_OPTIONS = {
    "round": (round, _options("RoundOptions", "ndigits", "round_mode")),
    "round_to_multiple": (round_to_multiple, _round_to_multiple_options),
    "round_binary": (round_binary, _options("RoundBinaryOptions", "round_mode")),
}


def _cumulative_options(name: str, options) -> dict:
    """CumulativeOptions' repr prints `start` as a pointer, so only an options object without a start can be read;
    one with a start needs the fields as a dict."""
    if not isinstance(options, dict) and "start=nullopt" not in str(options):
        raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: pass the CumulativeOptions fields as a dict "
                                          "(start, skip_nulls)")
    return _read_options(name, options, "CumulativeOptions", {"start": None, "skip_nulls": "skip_nulls"})


# The cumulative functions sit apart from _REGISTRY for the reason given above; tests/test_gpu_cumulative.py checks
# their options forms.
_CUMULATIVE_OPTIONS = {
    "cumulative_sum": (cumulative_sum, _cumulative_options),
    "cumulative_sum_checked": (cumulative_sum_checked, _cumulative_options),
    "cumulative_prod": (cumulative_prod, _cumulative_options),
    "cumulative_prod_checked": (cumulative_prod_checked, _cumulative_options),
    "cumulative_min": (cumulative_min, _cumulative_options),
    "cumulative_max": (cumulative_max, _cumulative_options),
    "cumulative_mean": (cumulative_mean, _cumulative_options),
}
_FUNCTIONS = {**_REGISTRY, **_STRING_TRANSFORM_OPTIONS, **_MATH_FUNCTIONS, **_MATH_OPTIONS, **_CUMULATIVE_OPTIONS}


def list_functions():
    return sorted(_FUNCTIONS)


def call_function(name: str, args: Sequence, options=None):
    """CallFunction(name, args, options): KeyError text follows registry.cc:95."""
    if name not in _FUNCTIONS:
        raise pa.ArrowKeyError(f"No function registered with name: {name}")
    fn, adapt = _FUNCTIONS[name]
    if options is None or adapt is None:
        return fn(*args)
    return fn(*args, **adapt(name, options))
