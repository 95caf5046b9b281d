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
from typing import Optional, Sequence, Union

import numpy as np
import pyarrow as pa

from . import _cabi as cabi
from .device import _NUMERIC as _NUMERIC_TYPES
from .device import Context, DeviceArray, arrow_type, check, type_id

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
    if s.is_valid:
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


def _prepare_binary(left: Operand, right: Operand):
    ctx = _ctx(left, right)
    ops = []
    ids = []
    for x in (left, right):
        if isinstance(x, DeviceArray):
            _require_numeric(x.type)
            ids.append(type_id(x.type))
            ops.append(x)
        else:
            s = _as_scalar(x)
            if pa.types.is_null(s.type):
                raise pa.ArrowNotImplementedError("null-typed scalar operands are not supported")
            _require_numeric(s.type)
            ids.append(type_id(s.type))
            ops.append(s)
    if not any(isinstance(o, DeviceArray) for o in ops):
        raise pa.ArrowNotImplementedError("arrow_b200: at least one operand must be a device array")
    tid = ids[0] if ids[0] == ids[1] and ids[0] in _NUMERIC_IDS else common_numeric(ids)
    keep = []  # keep ctypes structs alive for the call
    vals = []
    for o, i in zip(ops, ids):
        v = cabi.B2Value()
        if isinstance(o, DeviceArray):
            if i != tid:
                o = cast(o, arrow_type(tid))  # implicit safe cast
            c = o._c()
            keep.append((o, c))
            v.array = C.pointer(c)
            v.scalar = None
        else:
            sc = _scalar_to(o, tid)
            keep.append(sc)
            v.array = None
            v.scalar = C.pointer(sc)
        vals.append(v)
    return ctx, tid, vals, keep


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
    ctx = arr.ctx
    opt = cabi.B2CastOptions(dst, int(allow_int_overflow), int(allow_float_truncate), 0)
    cin, cout = arr._c(), cabi.B2Array()
    check(ctx.lib.b2_cast_numeric(ctx.handle, C.byref(cin), C.byref(opt), C.byref(cout), ctx.stream))
    return _out(ctx, cout, target_type)


def _arith(name: str, left: Operand, right: Operand) -> DeviceArray:
    ctx, tid, vals, keep = _prepare_binary(left, right)
    cout = cabi.B2Array()
    check(ctx.lib.b2_binary_arith(ctx.handle, cabi.ARITH_OPS[name], C.byref(vals[0]), C.byref(vals[1]),
                                  C.byref(cout), ctx.stream))
    return _out(ctx, cout, arrow_type(tid))


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
    ctx = lb.ctx
    cl, cout = lb._c(), cabi.B2Array()
    if isinstance(rb, DeviceArray):
        cr = rb._c()
        check(ctx.lib.b2_compare_binary(ctx.handle, cabi.COMPARE_OPS[name], C.byref(cl), C.byref(cr), None, 0, 1,
                                        C.byref(cout), ctx.stream))
    else:
        raw = rb.as_buffer().to_pybytes() if rb.is_valid else b""
        check(ctx.lib.b2_compare_binary(ctx.handle, cabi.COMPARE_OPS[name], C.byref(cl), None, raw, len(raw),
                                        int(rb.is_valid), C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.bool_())


def _compare(name: str, left: Operand, right: Operand) -> DeviceArray:
    if _binary_like(left) is not None or _binary_like(right) is not None:
        return _compare_binary(name, left, right)
    ctx, tid, vals, keep = _prepare_binary(left, right)
    cout = cabi.B2Array()
    check(ctx.lib.b2_compare(ctx.handle, cabi.COMPARE_OPS[name], C.byref(vals[0]), C.byref(vals[1]),
                             C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.bool_())


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
def _bool_value(x, keep):
    v = cabi.B2Value()
    if isinstance(x, DeviceArray):
        if not pa.types.is_boolean(x.type):
            raise pa.ArrowNotImplementedError(f"Function has no kernel matching input types ({x.type})")
        c = x._c()
        keep.append((x, c))
        v.array, v.scalar = C.pointer(c), None
    else:
        s = _as_scalar(x)
        if not (pa.types.is_boolean(s.type) or pa.types.is_null(s.type)):
            raise pa.ArrowNotImplementedError(f"Function has no kernel matching input types ({s.type})")
        sc = cabi.B2Scalar()
        sc.type, sc.is_valid = cabi.BOOL, 1 if s.is_valid else 0
        sc.bits = 1 if (s.is_valid and s.as_py()) else 0
        keep.append(sc)
        v.array, v.scalar = None, C.pointer(sc)
    return v


def _boolean(name: str, left, right=None) -> DeviceArray:
    ctx = _ctx(left, right)
    keep = []
    lv = _bool_value(left, keep)
    rv = _bool_value(right, keep) if name != "invert" else None
    cout = cabi.B2Array()
    check(ctx.lib.b2_boolean(ctx.handle, cabi.BOOLEAN_OPS[name], C.byref(lv), C.byref(rv) if rv is not None else None,
                             C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.bool_())


def and_(x, y): return _boolean("and", x, y)
def or_(x, y): return _boolean("or", x, y)
def xor(x, y): return _boolean("xor", x, y)
def and_not(x, y): return _boolean("and_not", x, y)
def and_kleene(x, y): return _boolean("and_kleene", x, y)
def or_kleene(x, y): return _boolean("or_kleene", x, y)
def and_not_kleene(x, y): return _boolean("and_not_kleene", x, y)
def invert(x): return _boolean("invert", x)


def _validity(name: str, arr: DeviceArray, nan_is_null: bool = False) -> DeviceArray:
    ctx = arr.ctx
    ca, cout = arr._c(), cabi.B2Array()
    check(ctx.lib.b2_validity(ctx.handle, cabi.VALIDITY_OPS[name], C.byref(ca), int(bool(nan_is_null)), C.byref(cout),
                              ctx.stream))
    return _out(ctx, cout, pa.bool_())


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
    cv = _bool_value(cond, keep)
    sides = [x if isinstance(x, DeviceArray) else _as_scalar(x) for x in (left, right)]
    types = [x.type for x in sides]
    if all(pa.types.is_boolean(t) or pa.types.is_null(t) for t in types):
        vals = [_bool_value(x, keep) for x in (left, right)]
        out_type = pa.bool_()
    else:
        for t in types:
            if pa.types.is_null(t):
                raise pa.ArrowNotImplementedError("null-typed scalar operands are not supported")
            _require_numeric(t)
        ids = [type_id(t) for t in types]
        tid = ids[0] if ids[0] == ids[1] else common_numeric(ids)
        out_type = arrow_type(tid)
        vals = []
        for x, i in zip(sides, ids):
            v = cabi.B2Value()
            if isinstance(x, DeviceArray):
                if i != tid:
                    x = cast(x, out_type)
                c = x._c()
                keep.append((x, c))
                v.array, v.scalar = C.pointer(c), None
            else:
                sc = _scalar_to(x, tid)
                keep.append(sc)
                v.array, v.scalar = None, C.pointer(sc)
            vals.append(v)
    cout = cabi.B2Array()
    check(ctx.lib.b2_if_else(ctx.handle, C.byref(cv), C.byref(vals[0]), C.byref(vals[1]), C.byref(cout), ctx.stream))
    return _out(ctx, cout, out_type)


# ------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------
def _null_selection(v) -> int:
    if v in ("drop", 0, None):
        return 0
    if v in ("emit_null", 1):
        return 1
    raise ValueError(f'"{v}" is not a valid null selection behavior')


def filter(values: DeviceArray, mask: DeviceArray, null_selection_behavior="drop") -> DeviceArray:
    """pyarrow.compute.filter / array_filter (kernels/vector_selection_filter_internal.cc:1043-1072)."""
    if not pa.types.is_boolean(mask.type):
        raise pa.ArrowNotImplementedError(
            f"Function 'array_filter' has no kernel matching input types ({values.type}, {mask.type})")
    if len(values) != len(mask):  # raised by the reference's VectorExecutor before the kernel runs
        raise pa.ArrowInvalid("Arguments for execution of vector kernel function 'array_filter' must all be the same length")
    ctx = values.ctx
    cv, cm, cout = values._c(), mask._c(), cabi.B2Array()
    check(ctx.lib.b2_filter(ctx.handle, C.byref(cv), C.byref(cm), _null_selection(null_selection_behavior),
                            C.byref(cout), ctx.stream))
    return _out(ctx, cout, values.type, values.dictionary)


def array_filter(values, mask, null_selection_behavior="drop"):
    return filter(values, mask, null_selection_behavior)


def filter_output_size(mask: DeviceArray, null_selection_behavior="drop") -> int:
    ctx = mask.ctx
    n = C.c_int64()
    cm = mask._c()
    check(ctx.lib.b2_filter_output_size(ctx.handle, C.byref(cm), _null_selection(null_selection_behavior),
                                        C.byref(n), ctx.stream))
    return n.value


def take_indices_from_filter(mask: DeviceArray, null_selection_behavior="drop") -> DeviceArray:
    """GetTakeIndices (kernels/vector_selection_take_internal.cc:298-305)."""
    ctx = mask.ctx
    cm, cout = mask._c(), cabi.B2Array()
    check(ctx.lib.b2_filter_indices(ctx.handle, C.byref(cm), _null_selection(null_selection_behavior),
                                    C.byref(cout), ctx.stream))
    return _out(ctx, cout, arrow_type(cout.type))


def take(values: DeviceArray, indices: DeviceArray, boundscheck: bool = True) -> DeviceArray:
    """pyarrow.compute.take / array_take (kernels/vector_selection_take_internal.cc:660-701)."""
    if not pa.types.is_integer(indices.type):
        raise pa.ArrowNotImplementedError(
            f"Function 'array_take' has no kernel matching input types ({values.type}, {indices.type})")
    ctx = values.ctx
    cv, ci, cout = values._c(), indices._c(), cabi.B2Array()
    check(ctx.lib.b2_take(ctx.handle, C.byref(cv), C.byref(ci), int(bool(boundscheck)), C.byref(cout),
                          ctx.stream))
    return _out(ctx, cout, values.type, values.dictionary)


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
    ctx = values.ctx
    keep = []
    ov = cabi.B2Value()
    co = other._c()
    keep.append(co)
    ov.array, ov.scalar = C.pointer(co), None
    cv, ci, cout = values._c(), indices._c(), cabi.B2Array()
    check(ctx.lib.b2_take_cast_arith(ctx.handle, C.byref(cv), C.byref(ci), type_id(target_type), cabi.ARITH_OPS[op], C.byref(ov),
                                     C.byref(cout), ctx.stream))
    return _out(ctx, cout, target_type)


def array_take(values, indices, boundscheck=True):
    return take(values, indices, boundscheck)


# ------------------------------------------------------------------------------------
# sort
# ------------------------------------------------------------------------------------
def _order(v) -> int:
    if v in ("ascending", 0):
        return 0
    if v in ("descending", 1):
        return 1
    raise ValueError(f'"{v}" is not a valid order')


def _placement(v) -> int:
    if v in ("at_start", 0):
        return 0
    if v in ("at_end", 1):
        return 1
    raise ValueError(f'"{v}" is not a valid null placement')


def array_sort_indices(arr: DeviceArray, order="ascending", null_placement="at_end") -> DeviceArray:
    """array_sort_indices (kernels/vector_array_sort.cc:524-540): stable argsort -> uint64."""
    ctx = arr.ctx
    ca, cout = arr._c(), cabi.B2Array()
    check(ctx.lib.b2_sort_indices(ctx.handle, C.byref(ca), _order(order), _placement(null_placement),
                                  C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.uint64())


def sort_payload(arr: DeviceArray, payload: DeviceArray, order="ascending", null_placement="at_end") -> DeviceArray:
    """stable sort of `arr` where row i carries payload[i] (uint32) instead of i: returns the payloads in sorted order
    (uint64) -- array_sort_indices followed by take(payload, indices), in the radix passes themselves"""
    ctx = arr.ctx
    ca, cp_, cout = arr._c(), payload._c(), cabi.B2Array()
    check(ctx.lib.b2_sort_payload(ctx.handle, C.byref(ca), C.byref(cp_), _order(order), _placement(null_placement),
                                  C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.uint64())


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
            orders.append(_order(o))
        ctx = cols[0].ctx
        cks = (cabi.B2Array * len(cols))(*[c._c() for c in cols])
        cor = (C.c_int32 * len(cols))(*orders)
        cout = cabi.B2Array()
        check(ctx.lib.b2_sort_indices_multi(ctx.handle, cks, len(cols), cor, _placement(null_placement), C.byref(cout), ctx.stream))
        return _out(ctx, cout, pa.uint64())
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
    ctx = arr.ctx
    ca, cout = arr._c(), cabi.B2Array()
    check(ctx.lib.b2_select_k(ctx.handle, C.byref(ca), int(k), _order(o), _placement(null_placement), C.byref(cout), ctx.stream))
    return _out(ctx, cout, pa.uint64())


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
    if mode == "only_valid":
        return pa.scalar(arr.length - nulls, pa.int64())
    if mode == "only_null":
        return pa.scalar(nulls, pa.int64())
    if mode == "all":
        return pa.scalar(arr.length, pa.int64())
    raise ValueError(f'"{mode}" is not a valid count mode')


# ------------------------------------------------------------------------------------
# unique / value_counts / dictionary_encode (kernels/vector_hash.cc:782-830)
# ------------------------------------------------------------------------------------
def _null_encoding(v) -> int:
    if v in ("mask", 0):
        return 0
    if v in ("encode", 1):
        return 1
    raise ValueError(f'"{v}" is not a valid null encoding behavior')


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
    if mode == "only_valid":
        return pa.scalar(len(u) - has_null, pa.int64())
    if mode == "only_null":
        return pa.scalar(has_null, pa.int64())
    if mode == "all":
        return pa.scalar(len(u), pa.int64())
    raise ValueError(f'"{mode}" is not a valid count mode')


def dictionary_encode(arr: DeviceArray, null_encoding="mask") -> DeviceArray:
    """dictionary_encode: int32 indices + dictionary (vector_hash.cc:173-232,826;
    DictionaryEncodeOptions api_vector.h:66-82)."""
    return _vector_hash(arr, _null_encoding(null_encoding), True, False)[0]


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
    if null_matching_behavior not in NULL_MATCHING:
        raise ValueError(f'"{null_matching_behavior}" is not a valid null matching behavior')
    return NULL_MATCHING[null_matching_behavior]


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
    cvs, h = value_set._c(), C.c_void_p()
    check(ctx.lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), nm, C.byref(h), ctx.stream))
    probe = ctx.lib.b2_index_in if index else ctx.lib.b2_is_in
    outs = []
    try:
        for c in chunks:  # the table is built once and probed per chunk
            if cast_to is not None:
                c = cast(c, cast_to, safe=True)
            cc, co = c._c(), cabi.B2Array()
            check(probe(h, C.byref(cc), C.byref(co), ctx.stream))
            outs.append(_out(ctx, co, pa.int32() if index else pa.bool_()))
    finally:
        ctx.lib.b2_set_lookup_destroy(h)
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
    ctx, cvs, h = value_set.ctx, value_set._c(), C.c_void_p()
    check(ctx.lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), NULL_MATCHING[null_matching_behavior], C.byref(h), ctx.stream))
    try:
        nbytes, shared = C.c_int64(), C.c_int32()
        check(ctx.lib.b2_set_lookup_table(h, C.byref(nbytes), C.byref(shared)))
        return nbytes.value, bool(shared.value)
    finally:
        ctx.lib.b2_set_lookup_destroy(h)


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
    raw = pattern.encode() if isinstance(pattern, str) else bytes(pattern)
    ctx, h = strings.ctx, C.c_void_p()
    is_utf8 = int(strings.type in _STRING_TYPES)
    check(ctx.lib.b2_string_match_create(ctx.handle, cabi.STRING_MATCH[name], raw, len(raw), is_utf8, C.byref(h), ctx.stream))
    try:
        cin, cout = strings._c(), cabi.B2Array()
        check(ctx.lib.b2_string_match(h, C.byref(cin), C.byref(cout), ctx.stream))
    finally:
        ctx.lib.b2_string_match_destroy(h)
    return _out(ctx, cout, pa.bool_())


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
    raw = pattern.encode() if isinstance(pattern, str) else bytes(pattern)
    ctx, h = Context.get(), C.c_void_p()
    check(ctx.lib.b2_string_match_create(ctx.handle, cabi.STRING_MATCH[kind], raw, len(raw), int(utf8), C.byref(h), ctx.stream))
    try:
        runs, nbytes = C.c_int32(), C.c_int64()
        check(ctx.lib.b2_string_match_info(h, C.byref(runs), C.byref(nbytes)))
        names = {v: k for k, v in cabi.STRING_MATCH.items()}
        return names[runs.value], nbytes.value
    finally:
        ctx.lib.b2_string_match_destroy(h)


def _match_options(name: str, options) -> dict:
    """MatchSubstringOptions as keywords: a dict {"pattern", "ignore_case"}, or pyarrow's MatchSubstringOptions (which
    exposes no attributes) read from its repr ('MatchSubstringOptions(pattern="ab", ignore_case=false)')."""
    if isinstance(options, dict):
        return dict(options)
    import re
    m = re.fullmatch(r'MatchSubstringOptions\(pattern="(.*)", ignore_case=(true|false)\)', str(options), re.S)
    if m is None:
        raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: pass the MatchSubstringOptions fields as a dict")
    return {"pattern": m.group(1), "ignore_case": m.group(2) == "true"}


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
        import re
        m = re.fullmatch(r"(\d\d):?(\d\d)", body) if len(body) in (4, 5) else None
        if m is None or (len(body) == 5 and body[2] != ":") or int(m.group(1)) > 23 or int(m.group(2)) > 59:
            raise pa.ArrowInvalid(f"Cannot locate or parse timezone '{tz}'")
        minutes = int(m.group(1)) * 60 + int(m.group(2))
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
    ctx = arr.ctx
    cin, cout = arr._c(), cabi.B2Array()
    check(ctx.lib.b2_temporal_field(ctx.handle, C.byref(cin), C.byref(desc), cabi.TEMPORAL_FIELDS[name], int(week_start),
                                    int(bool(count_from_zero)), C.byref(cout), ctx.stream))
    out_type = pa.bool_() if name == "is_leap_year" else pa.float64() if name == "subsecond" else pa.int64()
    return _out(ctx, cout, out_type)


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


_TEMPORAL_FIELDS = tuple(cabi.TEMPORAL_FIELDS)


def _day_of_week_options(options) -> dict:
    """DayOfWeekOptions as keywords: a dict, or pyarrow's DayOfWeekOptions (which exposes no attributes) read from its
    repr ('DayOfWeekOptions(count_from_zero=true, week_start=1)')."""
    if isinstance(options, dict):
        return dict(options)
    import re
    m = re.fullmatch(r"DayOfWeekOptions\(count_from_zero=(true|false), week_start=(-?\d+)\)", str(options))
    if m is None:
        raise pa.ArrowNotImplementedError("arrow_b200 day_of_week: pass the DayOfWeekOptions fields as a dict")
    return {"count_from_zero": m.group(1) == "true", "week_start": int(m.group(2))}


# ------------------------------------------------------------------------------------
# grouper + hash aggregates
# ------------------------------------------------------------------------------------
class Grouper:
    """arrow::compute::Grouper (compute/row/grouper.h:104-196) over fixed-width and utf8 / binary key columns."""

    def __init__(self, key_types: Sequence[pa.DataType], ctx: Optional[Context] = None):
        self.ctx = ctx or Context.get()
        self.key_types = [pa.lib.ensure_type(t) for t in key_types]
        ids = (C.c_int32 * len(self.key_types))(*[type_id(t) for t in self.key_types])
        h = C.c_void_p()
        check(self.ctx.lib.b2_grouper_create(self.ctx.handle, ids, len(self.key_types), C.byref(h)))
        self.handle = h

    def __del__(self):
        if getattr(self, "handle", None):
            self.ctx.lib.b2_grouper_destroy(self.handle)
            self.handle = None

    def _keys(self, keys):
        if isinstance(keys, DeviceArray):
            keys = [keys]
        if len(keys) != len(self.key_types):
            raise pa.ArrowInvalid(f"expected batch size {len(self.key_types)} but got {len(keys)}")
        for k, t in zip(keys, self.key_types):
            if k.type != t:
                raise pa.ArrowInvalid(f"expected batch value of type {t} but got {k.type}")
        carr = (cabi.B2Array * len(keys))(*[k._c() for k in keys])
        return carr

    def consume(self, keys) -> DeviceArray:
        carr, cout = self._keys(keys), cabi.B2Array()
        check(self.ctx.lib.b2_grouper_consume(self.handle, carr, C.byref(cout), self.ctx.stream))
        return _out(self.ctx, cout, pa.uint32())

    def lookup(self, keys) -> DeviceArray:
        carr, cout = self._keys(keys), cabi.B2Array()
        check(self.ctx.lib.b2_grouper_lookup(self.handle, carr, C.byref(cout), self.ctx.stream))
        return _out(self.ctx, cout, pa.uint32())

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


class HashAggregator:
    """One HashAggregateKernel state (compute/kernel.h:720-769): resize/consume/merge/finalize.

    hash_variance / hash_stddev take ddof=, hash_skew / hash_kurtosis take biased=; for these four min_count defaults
    to 0 (VarianceOptions / SkewOptions, api_aggregate.h:103-134), for the others to 1.  hash_list and hash_distinct
    (mode= as hash_count_distinct) finalize to a list<value_type>."""

    def __init__(self, function: str, value_type: Optional[pa.DataType], *, skip_nulls=True, min_count=None,
                 mode="only_valid", ddof=0, biased=True, ctx: Optional[Context] = None):
        self.ctx = ctx or Context.get()
        self.function = function
        self.value_type = value_type
        kind = cabi.HASH_AGG_KINDS[function]
        cm = {"only_valid": 0, "only_null": 1, "all": 2}[mode]
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
        h = C.c_void_p()
        check(self.ctx.lib.b2_hashagg_create(self.ctx.handle, kind, vt, C.byref(opts), C.byref(h)))
        self.handle = h

    def __del__(self):
        if getattr(self, "handle", None):
            self.ctx.lib.b2_hashagg_destroy(self.handle)
            self.handle = None

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
        cout = cabi.B2Array()
        check(self.ctx.lib.b2_hashagg_finalize(self.handle, C.byref(cout), self.ctx.stream))
        return _out(self.ctx, cout, arrow_type(cout.type))


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


class GroupBySumCount:
    """Fused consume of the aggregate node for `hash_sum` + `hash_count` over one value column
    (b2_groupby_sumcount_*): same results as Grouper + two HashAggregators."""

    def __init__(self, key_type, value_type, expected_groups=0, ctx: Optional[Context] = None):
        self.ctx = ctx or Context.get()
        self.key_type, self.value_type = pa.lib.ensure_type(key_type), pa.lib.ensure_type(value_type)
        h = C.c_void_p()
        check(self.ctx.lib.b2_groupby_sumcount_create(self.ctx.handle, type_id(self.key_type),
                                                      type_id(self.value_type), int(expected_groups), C.byref(h)))
        self.handle = h

    def __del__(self):
        if getattr(self, "handle", None):
            self.ctx.lib.b2_groupby_sumcount_destroy(self.handle)
            self.handle = None

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
_REGISTRY = {
    "cast": cast, "filter": filter, "array_filter": array_filter, "take": take, "array_take": array_take,
    "sort_indices": sort_indices, "array_sort_indices": array_sort_indices, "select_k_unstable": select_k_unstable,
    "if_else": if_else,
    "add": add, "subtract": subtract, "multiply": multiply, "divide": divide,
    "add_checked": add_checked, "subtract_checked": subtract_checked,
    "multiply_checked": multiply_checked, "divide_checked": divide_checked,
    "equal": equal, "not_equal": not_equal, "greater": greater, "greater_equal": greater_equal,
    "less": less, "less_equal": less_equal,
    "unique": unique, "value_counts": value_counts, "dictionary_encode": dictionary_encode, "count_distinct": count_distinct,
    "is_in": is_in, "index_in": index_in,
    "match_substring": match_substring, "starts_with": starts_with, "ends_with": ends_with, "match_like": match_like,
    "year": year, "month": month, "day": day, "day_of_year": day_of_year, "day_of_week": day_of_week, "quarter": quarter,
    "is_leap_year": is_leap_year, "hour": hour, "minute": minute, "second": second, "millisecond": millisecond,
    "microsecond": microsecond, "nanosecond": nanosecond, "subsecond": subsecond,
    "sum": sum, "mean": mean, "min_max": min_max, "min": min, "max": max, "count": count,
    "variance": variance, "stddev": stddev, "skew": skew, "kurtosis": kurtosis,
    "and": and_, "or": or_, "xor": xor, "and_not": and_not, "and_kleene": and_kleene, "or_kleene": or_kleene,
    "and_not_kleene": and_not_kleene, "invert": invert, "is_valid": is_valid, "is_null": is_null,
    "true_unless_null": true_unless_null, "is_nan": is_nan,
}


def list_functions():
    return sorted(_REGISTRY)


def _moment_options(options) -> dict:
    """ddof / skip_nulls / min_count (VarianceOptions) or skip_nulls / biased / min_count (SkewOptions) as keywords.  pyarrow
    exposes no attributes on those classes, so a non-dict is read from its repr ("VarianceOptions(ddof=1, skip_nulls=true,
    min_count=0)")."""
    if isinstance(options, dict):
        return dict(options)
    import re
    out = {}
    for key, value in re.findall(r"(\w+)=(-?\w+)", str(options)):
        out[key] = value == "true" if value in ("true", "false") else int(value)
    return out


def call_function(name: str, args: Sequence, options=None):
    """CallFunction(name, args, options): KeyError text follows registry.cc:95."""
    fn = _REGISTRY.get(name)
    if fn is None:
        raise pa.ArrowKeyError(f"No function registered with name: {name}")
    if options is None:
        return fn(*args)
    if name == "cast":
        return cast(args[0], options=options)
    if name in ("filter", "array_filter"):
        return fn(*args, null_selection_behavior=getattr(options, "null_selection_behavior", options))
    if name in ("take", "array_take"):
        return fn(*args, boundscheck=getattr(options, "boundscheck", True))
    if name == "array_sort_indices":
        return fn(*args, order=options.order, null_placement=options.null_placement)
    if name == "select_k_unstable":
        if isinstance(options, dict):
            return fn(*args, k=options["k"], sort_keys=options.get("sort_keys"))
        # pyarrow's SelectKOptions exposes no attributes: read k and the order from its repr
        # ("SelectKOptions(k=3, sort_keys=[FieldRef.Name(x) DESC])")
        import re
        text = str(options)
        return fn(*args, k=int(re.search(r"k=(-?\d+)", text).group(1)),
                  sort_keys=[("x", "descending" if " DESC" in text else "ascending")])
    if name == "dictionary_encode":
        return fn(*args, null_encoding=getattr(options, "null_encoding", options))
    if name in ("sum", "mean", "min_max", "min", "max"):
        return fn(*args, skip_nulls=options.skip_nulls, min_count=options.min_count)
    if name in ("variance", "stddev", "skew", "kurtosis"):
        return fn(*args, **_moment_options(options))
    if name in ("count", "count_distinct"):
        return fn(*args, mode=getattr(options, "mode", options))
    if name == "is_null":
        return fn(*args, nan_is_null=getattr(options, "nan_is_null", False))
    if name in ("is_in", "index_in"):
        # pyarrow's SetLookupOptions exposes no attributes and its repr cannot carry the value set: a dict is required
        if not isinstance(options, dict):
            raise pa.ArrowNotImplementedError(f"arrow_b200 {name}: pass the SetLookupOptions fields as a dict "
                                              "(value_set, skip_nulls, null_matching_behavior)")
        return fn(*args, **options)
    if name in ("match_substring", "starts_with", "ends_with", "match_like"):
        return fn(*args, **_match_options(name, options))
    if name == "day_of_week":
        return fn(*args, **_day_of_week_options(options))
    return fn(*args)
