"""An exact restatement of the numeric math functions, built without pyarrow.compute: abs, abs_checked, negate,
negate_checked, sign, sqrt, sqrt_checked, floor, ceil, trunc, bit_wise_not, power, power_checked, bit_wise_and / or /
xor, shift_left(_checked), shift_right(_checked), round, round_to_multiple and round_binary, with pyarrow 24's error
texts.

Values are Python lists (None = null).  Integers are Python ints wrapped to their type; floats are numpy float32 /
float64 scalars, so each operation is one IEEE operation of that type, as in the reference's C++ (RoundUtil::Pow10,
RoundImpl, Round::Call, RoundBinary::Call and RoundToMultiple::Call of kernels/scalar_round.cc; the op functors of
kernels/base_arithmetic_internal.h and kernels/scalar_arithmetic.cc).

An error is raised as MathError(kind, message), kind "Invalid" or "NotImplemented".  Where several rows fail, the
message is the last failing row's; a checked op checks valid rows only, unchecked power every row.
"""
import math

import numpy as np

INT_TYPES = ("int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64")
FLOAT_TYPES = ("float", "double")
NP_FLOAT = {"float": np.float32, "double": np.float64}
ROUND_MODES = ("down", "up", "towards_zero", "towards_infinity", "half_down", "half_up", "half_towards_zero",
               "half_towards_infinity", "half_to_even", "half_to_odd")
DIGITS10 = {"int8": 2, "uint8": 2, "int16": 4, "uint16": 4, "int32": 9, "uint32": 9, "int64": 18, "uint64": 19}


class MathError(Exception):
    def __init__(self, kind, message):
        super().__init__(message)
        self.kind, self.message = kind, message


def bits(t):
    return int(t.lstrip("u").removeprefix("int"))


def signed(t):
    return not t.startswith("u")


def lo_hi(t):
    b = bits(t)
    return (-(1 << (b - 1)), (1 << (b - 1)) - 1) if signed(t) else (0, (1 << b) - 1)


def wrap(v, t):
    b = bits(t)
    v &= (1 << b) - 1
    return v - (1 << b) if signed(t) and v >> (b - 1) else v


def _no_kernel(name, *types):
    raise MathError("NotImplemented", f"Function '{name}' has no kernel matching input types ({', '.join(types)})")


# ---------------------------------------------------------------------------------------------------------------------
# unary
# ---------------------------------------------------------------------------------------------------------------------
def _sign_bits(x, op):
    """x with its sign bit cleared ("abs") or flipped ("neg"), every other bit kept"""
    f = type(x)
    u, top = (np.uint32, 1 << 31) if f is np.float32 else (np.uint64, 1 << 63)
    raw = int(np.array([x], f).view(u)[0])
    raw = raw & ~top if op == "abs" else raw ^ top
    return np.array([raw], u).view(f)[0]


UNARY = ("abs", "abs_checked", "negate", "negate_checked", "sign", "sqrt", "sqrt_checked", "floor", "ceil", "trunc",
         "bit_wise_not")
TO_FLOAT = ("sqrt", "sqrt_checked", "floor", "ceil", "trunc")


def unary_out_type(name, t):
    if name in TO_FLOAT and t in INT_TYPES:
        return "double"
    if name == "sign" and t in INT_TYPES:
        return "int8"
    return t


def unary(name, values, t):
    """(values, output type) of unary function `name` over type t"""
    if (t in FLOAT_TYPES and name == "bit_wise_not") or (name == "negate_checked" and t in INT_TYPES and not signed(t)):
        _no_kernel(name, t)
    if name in TO_FLOAT and t in INT_TYPES:
        # the implicit safe cast to float64: a 64-bit integer beyond 2^53 may not be exact there
        lim = 1 << 53
        lo = -lim if signed(t) else 0
        for v in values:
            if bits(t) == 64 and v is not None and not lo <= v <= lim:
                raise MathError("Invalid", f"Integer value {v} not in range: {lo} to {lim}")
        values = [None if v is None else np.float64(v) for v in values]
        t = "double"
    out, err = [], None
    lo, hi = lo_hi(t) if t in INT_TYPES else (None, None)
    for v in values:
        if v is None:
            out.append(None)
            continue
        bad = False
        if t in FLOAT_TYPES:
            f = NP_FLOAT[t]
            v = f(v)
            with np.errstate(all="ignore"):
                if name in ("abs", "abs_checked"):
                    r = _sign_bits(v, "abs")
                elif name in ("negate", "negate_checked"):
                    r = _sign_bits(v, "neg")
                elif name == "sign":
                    r = v if np.isnan(v) else f(0) if v == 0 else f(-1) if np.signbit(v) else f(1)
                elif name == "sqrt":
                    r = f(np.nan) if v < 0 else np.sqrt(v)
                elif name == "sqrt_checked":
                    bad, r = v < 0, (v if v < 0 else np.sqrt(v))
                elif name == "floor":
                    r = np.floor(v)
                elif name == "ceil":
                    r = np.ceil(v)
                else:
                    r = np.trunc(v)
        else:
            if name in ("abs", "abs_checked"):
                bad = name == "abs_checked" and signed(t) and v == lo
                r = wrap(-v, t) if v < 0 else v
            elif name in ("negate", "negate_checked"):
                bad = name == "negate_checked" and v == lo
                r = wrap(-v, t)
            elif name == "sign":
                r = (v > 0) - (v < 0)
            else:
                r = wrap(~v, t)
        if bad:
            err = "square root of negative number" if name == "sqrt_checked" else "overflow"
        out.append(r)
    if err:
        raise MathError("Invalid", err)
    return out, unary_out_type(name, t)


# ---------------------------------------------------------------------------------------------------------------------
# binary integer ops
# ---------------------------------------------------------------------------------------------------------------------
BINARY = ("power", "power_checked", "bit_wise_and", "bit_wise_or", "bit_wise_xor", "shift_left", "shift_left_checked",
          "shift_right", "shift_right_checked")
NEGATIVE_POWER = "integers to negative integer powers are not allowed"
SHIFT_RANGE = "shift amount must be >= 0 and less than precision of type"


def _digits(t):
    """std::numeric_limits<T>::digits: the value bits, a signed type's sign bit excluded"""
    return bits(t) - (1 if signed(t) else 0)


def binary_one(name, l, r, t):
    """(result, error message or None) of one row; both operands of type t"""
    if name == "power":
        if r < 0:
            return 0, NEGATIVE_POWER
        base, e, p = l & (2 ** 64 - 1), r, 1
        while e:
            p = (p * (base if e & 1 else 1)) & (2 ** 64 - 1)
            base = (base * base) & (2 ** 64 - 1)
            e >>= 1
        return wrap(p, t), None
    if name == "power_checked":
        if r < 0:
            return 0, NEGATIVE_POWER
        if r == 0:
            return 1, None
        lo, hi = lo_hi(t)
        pw, overflow = 1, False
        for bit in bin(r)[2:]:
            p = pw * pw
            overflow |= not lo <= p <= hi
            pw = wrap(p, t)
            if bit == "1":
                p = pw * l
                overflow |= not lo <= p <= hi
                pw = wrap(p, t)
        return pw, "overflow" if overflow else None
    if name == "bit_wise_and":
        return l & r, None
    if name == "bit_wise_or":
        return l | r, None
    if name == "bit_wise_xor":
        return l ^ r, None
    out_of_range = r < 0 or r >= _digits(t)
    if out_of_range:
        return l, SHIFT_RANGE if name.endswith("_checked") else None
    if name.startswith("shift_left"):
        return wrap(l << r, t), None
    return l >> r, None  # Python's >> is arithmetic, a logical shift for a non-negative value


def binary(name, left, right, t, right_under_nulls=None):
    """values of binary op `name` over two lists (or a list and a scalar: a plain value, or None for a null scalar) of
    integer type t.  right_under_nulls: the right array's data buffer, null slots included (else 0 under a null)."""
    if t in FLOAT_TYPES:
        _no_kernel(name, t, t)
    n = len(left) if isinstance(left, list) else len(right)
    ls = left if isinstance(left, list) else [left] * n
    rs = right if isinstance(right, list) else [right] * n
    if (not isinstance(left, list) and left is None) or (not isinstance(right, list) and right is None):
        return [None] * n
    out, err = [], None
    under = right_under_nulls or [0] * n
    for l, r, u in zip(ls, rs, under):
        valid = l is not None and r is not None
        lv = 0 if l is None else l
        rv = u if r is None else r
        res, e = binary_one(name, lv, rv, t)
        # unchecked power is a plain ScalarBinary: every slot is computed and checked, a null one's value being what
        # its buffer holds (tests give it explicitly)
        if e and (valid or name == "power"):
            err = e
        out.append(res if valid else None)
    if err:
        raise MathError("Invalid", err)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# rounding
# ---------------------------------------------------------------------------------------------------------------------
_LUT = [np.float64(np.float32(10.0 ** k)) for k in range(16)]  # the float literals 1e0F .. 1e15F, as doubles


def pow10(power):
    """RoundUtil::Pow10<double>(power)"""
    a = builtin_abs(power)
    p = _LUT[min(a, 15)]
    k = a - 15
    with np.errstate(over="ignore"):
        while k > 0 and np.isfinite(p):
            p = p * np.float64(10.0)
            k -= 1
    with np.errstate(divide="ignore"):
        return p if power >= 0 else np.float64(1.0) / p


builtin_abs = abs


def _std_round(v):
    """std::round: half away from zero, exact"""
    f = type(v)
    t = np.trunc(v)
    return t + f(np.copysign(1.0, v)) if builtin_abs(v - t) >= f(0.5) else t


def _round_mode_float(v, mode):
    f = type(v)
    if mode in ("down", "half_down"):
        return np.floor(v)
    if mode in ("up", "half_up"):
        return np.ceil(v)
    if mode in ("towards_zero", "half_towards_zero"):
        return np.trunc(v)
    if mode in ("towards_infinity", "half_towards_infinity"):
        return np.floor(v) if np.signbit(v) else np.ceil(v)
    if mode == "half_to_even":
        return _std_round(v * f(0.5)) * f(2)
    return np.floor(v * f(0.5)) + np.ceil(v * f(0.5))


OVERFLOW_ROUNDING = "overflow occurred during rounding"


def round_float(arg, p, scale_mul, unscale_div, mode):
    """(value, failed) of Round / RoundToMultiple / RoundBinary::Call on a float, in arg's own type"""
    with np.errstate(all="ignore"):
        if not np.isfinite(arg):
            return arg, False
        r = arg * p if scale_mul else arg / p
        frac = r - np.floor(r)
        if frac == 0:
            return arg, False
        r = _std_round(r) if mode.startswith("half") and frac != 0.5 else _round_mode_float(r, mode)
        r = r / p if unscale_div else r * p
        if not np.isfinite(r):
            return arg, True
        return r, False


def round_int(arg, multiple, t, mode):
    """(value, error message or None) of RoundToMultiple<integer>::Call"""
    lo, hi = lo_hi(t)
    q = builtin_abs(arg) // multiple * (1 if arg >= 0 else -1)
    floor = q * multiple
    rem = builtin_abs(arg - floor)
    if rem == 0:
        return arg, None
    # remainder * 2: in int for the types narrower than int, wrapping in T for the others
    twice = rem * 2 if bits(t) < 32 else wrap(rem * 2, t)

    def fail(direction, plural):
        return arg, f"Rounding {arg} {direction} to multiple{'s' if plural else ''} of {multiple} would overflow"

    if mode.startswith("half") and twice != multiple:
        if twice > multiple:
            if arg >= 0:
                return fail("up", True) if hi - multiple < floor else (floor + multiple, None)
            return fail("down", True) if lo + multiple > floor else (floor - multiple, None)
        return floor, None
    m = mode
    if mode == "half_to_even":
        if q % 2 == 0:
            return floor, None
        m = "towards_infinity"
    elif mode == "half_to_odd":
        if q % 2 != 0:
            return floor, None
        m = "towards_infinity"
    else:
        m = mode.removeprefix("half_")
    if m in ("down", "towards_infinity") and signed(t) and arg < 0:
        return fail("down", False) if lo + multiple > floor else (floor - multiple, None)
    if m in ("up", "towards_infinity") and arg > 0:
        return fail("up", False) if hi - multiple < floor else (floor + multiple, None)
    if m == "towards_infinity" and not signed(t):
        return floor + multiple, None
    return floor, None


def _finish(out, err):
    if err:
        raise MathError("Invalid", err)
    return out


def round_(values, t, ndigits=0, mode="half_to_even"):
    if t in INT_TYPES:
        if -ndigits > DIGITS10[t]:
            raise MathError("Invalid", f"Rounding to {ndigits} digits is out of range for type {t}")
        if ndigits >= 0:
            return list(values)
        return round_to_multiple(values, t, 10 ** -ndigits, mode)
    f = NP_FLOAT[t]
    with np.errstate(over="ignore"):
        p = f(pow10(builtin_abs(ndigits)))
    out, err = [], None
    for v in values:
        if v is None:
            out.append(None)
            continue
        r, failed = round_float(f(v), p, ndigits >= 0, ndigits > 0, mode)
        err = OVERFLOW_ROUNDING if failed else err
        out.append(r)
    return _finish(out, err)


def round_to_multiple(values, t, multiple, mode="half_to_even"):
    """multiple: already of type t (the caller applies the safe cast), and positive"""
    out, err = [], None
    for v in values:
        if v is None:
            out.append(None)
            continue
        if t in INT_TYPES:
            r, e = round_int(v, multiple, t, mode)
            err = e or err
        else:
            f = NP_FLOAT[t]
            r, failed = round_float(f(v), f(multiple), False, False, mode)
            err = OVERFLOW_ROUNDING if failed else err
        out.append(r)
    return _finish(out, err)


def round_binary(values, t, digits, mode="half_to_even"):
    """digits: a list of int32 (or None), or one int32 / None for a scalar"""
    n = len(values) if isinstance(values, list) else len(digits)
    xs = values if isinstance(values, list) else [values] * n
    ds = digits if isinstance(digits, list) else [digits] * n
    if (not isinstance(values, list) and values is None) or (not isinstance(digits, list) and digits is None):
        return [None] * n
    out, err = [], None
    for v, s in zip(xs, ds):
        if v is None or s is None:
            out.append(None)
            continue
        if t in INT_TYPES:
            if s >= 0:
                out.append(v)
                continue
            if -s > DIGITS10[t] or s == -(1 << 31):
                err = f"Rounding to {s} digits is out of range for type {t}"
                out.append(v)
                continue
            r, e = round_int(v, 10 ** -s, t, mode)
            err = e or err
            out.append(r)
        else:
            f = NP_FLOAT[t]
            a = s if s >= 0 else wrap(-s, "int32")  # std::abs of an int32: INT32_MIN stays negative
            r, failed = round_float(np.float64(f(v)), pow10(a), s >= 0, s > 0, mode)
            err = OVERFLOW_ROUNDING if failed else err
            with np.errstate(over="ignore"):
                out.append(f(v) if failed else f(r))
    return _finish(out, err)
