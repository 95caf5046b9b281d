"""Exact references for the element-wise kernels: cast, arithmetic, comparison, if_else and the fused take + cast + arithmetic.

Nothing here relies on a CPU float behaviour beyond IEEE double: integers are Python ints, float64 arithmetic is the exact
`Fraction` result rounded by `round_rational` (nearest-even, with the overflow, subnormal and signed-zero rules), float32
arithmetic is one double operation rounded once to float32 -- exact for + - * /, since 53 >= 2 * 24 + 2 -- and every
int -> float conversion rounds the exact integer.  Error texts are the reference's, and for checked arithmetic the error is
that of the LAST offending valid row: the reference's applicator (ScalarBinaryNotNullStateful) runs every row and each
failing row overwrites the status, so `divide_checked` of [INT_MIN, 5] / [-1, 0] says "divide by zero".

Results are compared with exact_ref.assert_same: bit-exact on valid slots, any NaN equal to any NaN (the payload of an
arithmetic NaN is implementation-defined)."""
import math
from fractions import Fraction

import numpy as np
import pyarrow as pa

INT_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()]
FLOAT_TYPES = [pa.float32(), pa.float64()]
NUMERIC = INT_TYPES + FLOAT_TYPES
ARITH_OPS = ("add", "subtract", "multiply", "divide", "add_checked", "subtract_checked", "multiply_checked", "divide_checked")
COMPARE_OPS = ("equal", "not_equal", "greater", "greater_equal", "less", "less_equal")

# (mantissa bits incl. the implicit one, minimum normal exponent, maximum exponent)
_FMT = {32: (24, -126, 127), 64: (53, -1022, 1023)}


def np_dtype(t: pa.DataType):
    return np.dtype(t.to_pandas_dtype())


def int_range(t: pa.DataType):
    info = np.iinfo(np_dtype(t))
    return int(info.min), int(info.max)


def wrap(x: int, t: pa.DataType) -> int:
    """x reduced mod 2^w into the integer type t"""
    lo, _ = int_range(t)
    w = t.bit_width
    return ((x - lo) % (1 << w)) + lo


F32_MAX = float(np.finfo(np.float32).max)
F64_MAX = float(np.finfo(np.float64).max)


def f32_bits(u: int) -> float:
    return float(np.array([u], np.uint32).view(np.float32)[0])


def f64_bits(u: int) -> float:
    return float(np.array([u], np.uint64).view(np.float64)[0])


# ---------------------------------------------------------------------------------------------------------------------
# edge values shared by the element-wise and sort tests
# ---------------------------------------------------------------------------------------------------------------------
def int_edges(t: pa.DataType) -> list:
    """min, min + 1, -1, 0, 1, max - 1, max, +-2^(w/2) and neighbours, and factors whose products land near 2^(w-1)"""
    lo, hi = int_range(t)
    w = t.bit_width
    h = 1 << (w // 2)
    cand = [lo, lo + 1, -1, 0, 1, 2, 3, hi - 1, hi, h, -h, h - 1, h + 1, -h - 1, h // 2, -(h // 2), hi // 2, hi // 2 + 1,
            hi // 3, lo // 2, -(hi // 3), 7]
    return sorted({v for v in cand if lo <= v <= hi})


def float_edges(t: pa.DataType) -> list:
    """+-0, +-inf, NaNs of several payloads, subnormals, the largest finite value, values whose sums / quotients are ties
    and values that overflow when doubled"""
    from tests.exact_ref import F32_SPECIAL, F64_SPECIAL
    if t == pa.float32():
        sp = [f32_bits(b) for b in F32_SPECIAL.values() if b != 0x7F800001]   # a signalling NaN becomes quiet in a double
        p, mx = 24, F32_MAX
    else:
        sp = [f64_bits(b) for b in F64_SPECIAL.values()]
        p, mx = 53, F64_MAX
    tiny = float(np.finfo(t.to_pandas_dtype()).smallest_subnormal)
    normal = float(np.finfo(t.to_pandas_dtype()).tiny)
    return sp + [tiny * 3, normal, normal - tiny, -normal, mx, -mx, mx / 2, 1.0, -1.0, 1.5, 3.0, 0.1 if t == pa.float64() else
                 float(np.float32(0.1)), float(2 ** p), float(2 ** p + 2), 2.0 ** -p, 1.0 + 2.0 ** (1 - p), 7.0]


def edges(t: pa.DataType) -> list:
    return int_edges(t) if pa.types.is_integer(t) else float_edges(t)


# ---------------------------------------------------------------------------------------------------------------------
# rounding
# ---------------------------------------------------------------------------------------------------------------------
def round_rational(q, width: int, negative_zero=False) -> float:
    """the exact rational q rounded to nearest-even in IEEE binary32 (width 32) or binary64, as a Python float (a binary32
    value is exactly representable in a double).  Overflow gives +-inf; a result that underflows to zero keeps q's sign; an
    exact zero is -0.0 when `negative_zero`."""
    q = Fraction(q)
    if q == 0:
        return -0.0 if negative_zero else 0.0
    p, emin, emax = _FMT[width]
    neg = q < 0
    a = -q if neg else q
    e = a.numerator.bit_length() - a.denominator.bit_length()   # 2^e <= a < 2^(e+1) after the correction
    if Fraction(2) ** e > a:
        e -= 1
    qe = max(e, emin) - (p - 1)                                  # exponent of the last mantissa bit (fixed when subnormal)
    scaled = a / Fraction(2) ** qe
    m = scaled.numerator // scaled.denominator
    rem = scaled - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m & 1):
        m += 1
    if m and m.bit_length() + qe > emax + 1:                     # m * 2^qe >= 2^(emax+1)
        r = math.inf
    else:
        r = math.ldexp(m, qe)
    return -r if neg else r


def f64_to_f32(x: float) -> float:
    """float64 -> float32, round to nearest-even (NaN stays NaN, the sign of zeros and infinities is kept)"""
    if math.isnan(x) or math.isinf(x):
        return x
    return round_rational(Fraction(x), 32, negative_zero=math.copysign(1.0, x) < 0)


def int_to_float(v: int, width: int) -> float:
    """an integer rounded once (nearest-even) to float32 / float64 -- never through a double first"""
    return round_rational(v, width)


def to_array(vals, t: pa.DataType, valid=None) -> pa.Array:
    """a list of Python ints / floats (floats already representable in t) as an Arrow array of t; nothing is rounded"""
    dt = np_dtype(t)
    if pa.types.is_integer(t):
        raw = np.array([int(v) for v in vals], dtype=object).astype(dt) if len(vals) else np.zeros(0, dt)
    else:
        raw = np.array(vals, dtype=np.float64).astype(dt)
        assert all(math.isnan(a) and math.isnan(b) or a == b for a, b in zip(raw.astype(np.float64).tolist(), vals)), \
            "to_array: a value is not representable in the target type"
    mask = None if valid is None else ~np.asarray(valid, bool)
    return pa.array(raw, type=t, mask=mask)


def pylist(arr: pa.Array) -> list:
    """every slot's value as a Python int / float, nulls included (whatever the buffer holds there)"""
    from tests.exact_ref import raw
    return raw(arr).tolist()


# ---------------------------------------------------------------------------------------------------------------------
# casts
# ---------------------------------------------------------------------------------------------------------------------
def safe_int_range(src: pa.DataType, dst: pa.DataType):
    """the range a safe cast of integer type src to dst admits, in src (GetSafeMinMax for int -> int; the 2^24 / 2^53 bound
    for int -> float where the source can exceed it), or None when every src value passes"""
    lo, hi = int_range(src)
    if pa.types.is_integer(dst):
        dlo, dhi = int_range(dst)
        r = (max(lo, dlo), min(hi, dhi))
    else:
        if src.bit_width < 32 or (src.bit_width == 32 and dst == pa.float64()):
            return None
        limit = 1 << (24 if dst == pa.float32() else 53)
        r = (max(lo, -limit if pa.types.is_signed_integer(src) else 0), min(hi, limit))
    return None if r == (lo, hi) else r


def c_float_text(x: float) -> str:
    """printf("%f") of a double, as the reference's std::to_string spells it ("-nan" for a NaN with the sign bit)"""
    if math.isnan(x):
        return "-nan" if math.copysign(1.0, x) < 0 else "nan"
    return f"{x:f}"


def _cvtt32(x: float) -> int:
    return math.trunc(x) if -2147483649.0 < x < 2147483648.0 else -(1 << 31)


def _cvtt64(x: float) -> int:
    return math.trunc(x) if -9223372036854775808.0 <= x < 9223372036854775808.0 else -(1 << 63)


def float_to_int_unsafe(x: float, dst: pa.DataType) -> int:
    """float -> int with safe=False, as scalar_cast.cu convert() defines it for every input -- out of range, +-inf and NaN
    included: x86's cvttsd2si / cvttss2si, whose out-of-range answer is the "integer indefinite" value INT_MIN of the
    instruction's width, narrowed to the target; uint64 subtracts 2^63 first for x >= 2^63 (the compilers' sequence)"""
    w = dst.bit_width
    if dst == pa.int64():
        return _cvtt64(x)
    if dst == pa.uint64():
        if x >= 9223372036854775808.0:   # x - 2^63 is exact below 2^64 and stays >= 2^63 above it
            return (_cvtt64(x - 9223372036854775808.0) % (1 << 64)) ^ (1 << 63)
        return _cvtt64(x) % (1 << 64)
    if dst == pa.uint32():
        return _cvtt64(x) % (1 << 32)
    return wrap(_cvtt32(x), dst) if w < 32 else _cvtt32(x)


def cast_value(x, src: pa.DataType, dst: pa.DataType, safe: bool):
    """one valid value: (result, None) or (None, the reference's error text)"""
    if pa.types.is_integer(src):
        x = int(x)
        if safe:
            r = safe_int_range(src, dst)
            if r is not None and not r[0] <= x <= r[1]:
                return None, f"Integer value {x} not in range: {r[0]} to {r[1]}"
        if pa.types.is_integer(dst):
            return wrap(x, dst), None
        return int_to_float(x, dst.bit_width), None
    x = float(x)
    if pa.types.is_floating(dst):
        return (f64_to_f32(x) if dst == pa.float32() else x), None
    if safe:
        lo, hi = int_range(dst)
        if not math.isfinite(x) or x != math.trunc(x) or not lo <= x <= hi:
            return None, f"Float value {c_float_text(x)} was truncated converting to {dst}"
    return float_to_int_unsafe(x, dst), None


def cast(arr: pa.Array, dst: pa.DataType, safe: bool = True) -> pa.Array:
    """the exact cast; raises pa.ArrowInvalid naming the first offending valid row, as the reference does"""
    from tests.exact_ref import valid_mask
    src = arr.type
    valid = valid_mask(arr)
    out = []
    for x, ok in zip(pylist(arr), valid):
        y, err = cast_value(x, src, dst, safe and ok)
        if err is not None and ok:
            raise pa.ArrowInvalid(err)
        if y is None:
            y = 0
        out.append(y)
    return to_array(out, dst, valid if arr.null_count else None)


# ---------------------------------------------------------------------------------------------------------------------
# dispatch: CommonNumeric and the implicit safe cast of the operands
# ---------------------------------------------------------------------------------------------------------------------
def common_numeric(types):
    if pa.float64() in types:
        return pa.float64()
    if pa.float32() in types:
        return pa.float32()
    ms = max([t.bit_width for t in types if pa.types.is_signed_integer(t)], default=0)
    mu = max([t.bit_width for t in types if pa.types.is_unsigned_integer(t)], default=0)
    if ms == 0:
        return {8: pa.uint8(), 16: pa.uint16(), 32: pa.uint32()}.get(mu, pa.uint64())
    if ms <= mu:
        ms = 1 << mu.bit_length()
    return {8: pa.int8(), 16: pa.int16(), 32: pa.int32()}.get(ms, pa.int64())


def operand(x, n: int):
    """(type, Python values, valid) of an array or a scalar broadcast to n rows"""
    from tests.exact_ref import valid_mask
    if isinstance(x, pa.Array):
        return x.type, pylist(x), valid_mask(x)
    if not x.is_valid:
        return x.type, [0] * n, np.zeros(n, bool)
    return x.type, [x.as_py()] * n, np.ones(n, bool)


def promote(x, t: pa.DataType, n: int):
    """operand x safely cast to t -> (values, valid); raises the reference's ArrowInvalid for an operand that does not fit"""
    xt, vals, valid = operand(x, n)
    if xt == t:
        return vals, valid
    if isinstance(x, pa.Scalar):
        if not x.is_valid:
            return vals, valid
        y, err = cast_value(vals[0], xt, t, True)
        if err is not None:
            raise pa.ArrowInvalid(err)
        return [y] * n, valid
    return pylist(cast(x, t, True)), valid


def _length(*xs):
    return next(len(x) for x in xs if isinstance(x, pa.Array))


def _types(*xs):
    return [x.type for x in xs]


# ---------------------------------------------------------------------------------------------------------------------
# arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def _trunc_div(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def int_op(op: str, a: int, b: int, t: pa.DataType):
    """(result, error kind or None) of one valid integer row"""
    base, checked = op.replace("_checked", ""), op.endswith("_checked")
    lo, hi = int_range(t)
    if base == "divide":
        if b == 0:
            return 0, "divide by zero"
        exact = _trunc_div(a, b)
        if not lo <= exact <= hi:                    # INT_MIN / -1
            return (a, "overflow") if checked else (0, None)
        return exact, None
    exact = {"add": a + b, "subtract": a - b, "multiply": a * b}[base]
    if checked and not lo <= exact <= hi:
        return wrap(exact, t), "overflow"
    return wrap(exact, t), None


def _f64_exact(base: str, a: float, b: float) -> float:
    """one float64 operation: the exact result rounded once; non-finite operands, x / 0 and 0 / 0 by IEEE's rules (which
    any double unit computes exactly)"""
    if not (math.isfinite(a) and math.isfinite(b)) or (base == "divide" and b == 0):
        with np.errstate(all="ignore"):
            return float({"add": np.add, "subtract": np.subtract, "multiply": np.multiply,
                          "divide": np.divide}[base](np.float64(a), np.float64(b)))
    A, B = Fraction(a), Fraction(b)
    sa, sb = math.copysign(1.0, a) < 0, math.copysign(1.0, b) < 0
    if base == "add":
        q, negz = A + B, sa and sb
    elif base == "subtract":
        q, negz = A - B, sa and not sb
    elif base == "multiply":
        q, negz = A * B, sa != sb
    else:
        q, negz = A / B, sa != sb
    return round_rational(q, 64, negative_zero=negz)


def float_op(op: str, a: float, b: float, t: pa.DataType):
    base, checked = op.replace("_checked", ""), op.endswith("_checked")
    if base == "divide" and checked and b == 0:
        return 0.0, "divide by zero"
    if t == pa.float64():
        return _f64_exact(base, a, b), None
    with np.errstate(all="ignore"):   # float32: one double operation, rounded once (exact: 53 >= 2 * 24 + 2)
        d = float({"add": np.add, "subtract": np.subtract, "multiply": np.multiply,
                   "divide": np.divide}[base](np.float64(a), np.float64(b)))
    return f64_to_f32(d), None


def arithmetic(op: str, left, right) -> pa.Array:
    """op(left, right) with the reference's dispatch; raises pa.ArrowInvalid like the reference"""
    n = _length(left, right)
    t = _types(left, right)
    t = t[0] if t[0] == t[1] else common_numeric(t)
    # the operands are cast first: an array that does not fit raises even beside a null scalar
    (a, va), (b, vb) = promote(left, t, n), promote(right, t, n)
    valid = va & vb
    fn = int_op if pa.types.is_integer(t) else float_op
    out, last = [], None
    for x, y, ok in zip(a, b, valid):
        r, err = fn(op, x, y, t)
        if err is not None and ok:
            last = err
        out.append(r)
    if last is not None:
        raise pa.ArrowInvalid(last)
    return to_array(out, t, valid)


# ---------------------------------------------------------------------------------------------------------------------
# comparison and if_else
# ---------------------------------------------------------------------------------------------------------------------
_CMP = {"equal": lambda x, y: x == y, "not_equal": lambda x, y: x != y, "greater": lambda x, y: x > y,
        "greater_equal": lambda x, y: x >= y, "less": lambda x, y: x < y, "less_equal": lambda x, y: x <= y}


def compare(op: str, left, right) -> pa.Array:
    """IEEE comparison of the promoted operands: a NaN is unequal to everything (itself included), -0.0 == +0.0; exact on
    integers (Python ints)"""
    n = _length(left, right)
    t = _types(left, right)
    t = t[0] if t[0] == t[1] else common_numeric(t)
    (a, va), (b, vb) = promote(left, t, n), promote(right, t, n)
    valid = va & vb
    out = [bool(_CMP[op](x, y)) for x, y in zip(a, b)]
    return pa.array(out, pa.bool_(), mask=~valid)


def if_else(cond, left, right) -> pa.Array:
    """cond ? left : right after the safe promotion to CommonNumeric; valid = cond valid AND the chosen side's validity.  A
    selection: every selected value comes through bit for bit, NaN payloads and -0.0 included (a float64 NaN is kept as its
    bits, never rebuilt from a Python float)"""
    from tests.exact_ref import raw, valid_mask
    n = _length(cond, left, right)
    t = _types(left, right)
    t = t[0] if t[0] == t[1] else common_numeric(t)
    dt = np_dtype(t)
    if isinstance(cond, pa.Array):
        c, vc = raw(cond.cast(pa.uint8())).astype(bool), valid_mask(cond)
    else:
        c, vc = np.full(n, bool(cond.as_py()) if cond.is_valid else False), np.full(n, cond.is_valid)
    cols = []
    for x in (left, right):
        if isinstance(x, pa.Scalar) and not x.is_valid:
            cols.append((np.zeros(n, dt), np.zeros(n, bool)))
        elif x.type != t:
            vals, ok = promote(x, t, n)
            cols.append((raw(to_array(vals, t)), ok))
        elif isinstance(x, pa.Array):
            cols.append((raw(x), valid_mask(x)))
        else:
            cols.append((np.frombuffer(_scalar_bytes(x), dt).repeat(n), np.ones(n, bool)))
    (l, vl), (r, vr) = cols
    valid = vc & np.where(c, vl, vr)
    return pa.Array.from_buffers(t, n, [pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()),
                                        pa.py_buffer(np.where(c, l, r).astype(dt).tobytes())], null_count=int((~valid).sum()))


def _scalar_bytes(s: pa.Scalar) -> bytes:
    """the value bytes of a valid fixed-width scalar"""
    a = pa.array([s], s.type)
    return a.buffers()[1].to_pybytes()[:s.type.bit_width // 8]


# ---------------------------------------------------------------------------------------------------------------------
# fused take + cast + arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def take_cast_arith(values: pa.Array, indices: pa.Array, to: pa.DataType, op: str, other) -> pa.Array:
    """op(cast(take(values, indices), to, safe=False), other): each taken value converted exactly (float64 -> float32 and
    int -> float round once to nearest-even), then one IEEE operation; valid = index valid AND value valid AND other valid"""
    from tests.exact_ref import valid_mask
    idx, iv = pylist(indices), valid_mask(indices)
    vals, vv = pylist(values), valid_mask(values)
    n = len(indices)
    ot, ovals, ov = operand(other, n)
    assert ot == to
    out, valid = [], np.zeros(n, bool)
    for i in range(n):
        if not iv[i]:
            out.append(0.0)
            continue
        j = idx[i]
        x, _ = cast_value(vals[j], values.type, to, False)
        r, _ = float_op(op, x, ovals[i], to)
        out.append(r)
        valid[i] = vv[j] and ov[i]
    return to_array(out, to, valid)
