"""CPU: the exact element-wise references (tests/elementwise_ref.py) and the oracle's cast / arithmetic / compare / if_else
against the reference binary (pyarrow) on full-range integers, NaN, +-0, +-inf, subnormals and rounding edges, over every
type pair in the array / array, array / scalar and scalar / array shapes -- the references the GPU tests in
test_gpu_elementwise_edges.py hold the kernels to.  Also: the implicit safe cast of scalar operands (compute._scalar_to,
which needs no device), and the float -> uint32 cases where the reference disagrees with itself."""
import itertools
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200.device import type_id
from oracle import arrow_oracle as ora
from tests import elementwise_ref as ew
from tests import exact_ref as er
from tests.elementwise_ref import F32_MAX, edges, f32_bits, float_edges

def tame(t: pa.DataType) -> list:
    """small values no checked op overflows on (zeros excluded: the divisions must not fail either)"""
    vals = [1, 2, 3, 5, 7] + ([-1, -2, -6] if not pa.types.is_unsigned_integer(t) else [4, 6, 9])
    if pa.types.is_floating(t):
        vals = [float(v) for v in vals] + [0.5, -0.0, 0.25]
    return vals


def pair_arrays(tl, tr, vl, vr):
    """the cartesian product of two value lists as two equal-length arrays, every fifth row null on one side"""
    rows = list(itertools.product(vl, vr))
    n = len(rows)
    a = ew.to_array([r[0] for r in rows], tl, np.arange(n) % 5 != 3)
    b = ew.to_array([r[1] for r in rows], tr, np.arange(n) % 7 != 4)
    return a, b


def outcome(fn):
    """("ok", result) or (exception type, text)"""
    try:
        return "ok", fn()
    except (pa.ArrowInvalid, pa.ArrowNotImplementedError, OverflowError) as e:
        return type(e).__name__, str(e)


def same_result(got: pa.Array, want: pa.Array, msg=""):
    """exact_ref.assert_same, and for boolean results the values of the valid slots and the validity"""
    if isinstance(want, pa.ChunkedArray):
        want = want.combine_chunks()
    if pa.types.is_boolean(want.type):
        assert got.type == want.type and got.to_pylist() == want.to_pylist(), f"{msg}: {got.to_pylist()} != {want.to_pylist()}"
    else:
        er.assert_same(got, want, msg=msg)


def same_outcome(got, want, msg):
    assert got[0] == want[0], f"{msg}: got {got[0]} {got[1] if got[0] != 'ok' else ''} want {want[0]} {want[1] if want[0] != 'ok' else ''}"
    if got[0] == "ok":
        same_result(got[1], want[1], msg)
    else:
        assert got[1] == want[1], f"{msg}: {got[1]!r} != {want[1]!r}"


def scalars(t):
    v = edges(t)
    return [pa.scalar(x, t) for x in (v[0], v[len(v) // 2], v[-1])] + [pa.scalar(None, t)]


SHAPES = ("array_array", "array_scalar", "scalar_array")


def operands(shape, tl, tr, vl, vr):
    a, b = pair_arrays(tl, tr, vl, vr)
    if shape == "array_array":
        return [(a, b)]
    if shape == "array_scalar":
        return [(a, s) for s in scalars(tr)]
    return [(s, b) for s in scalars(tl)]


# ---------------------------------------------------------------------------------------------------------------------
# the reference helpers themselves
# ---------------------------------------------------------------------------------------------------------------------
def test_round_rational_f32_edges():
    ulp_max = 2.0 ** (127 - 23)
    cases = [
        (1 + 2.0 ** -24, 1.0),                          # tie: to the even mantissa
        (1 + 3 * 2.0 ** -24, 1 + 2.0 ** -22),           # tie: up to the even neighbour
        (1 + 2.0 ** -24 + 2.0 ** -40, 1 + 2.0 ** -23),  # above the tie
        (F32_MAX + ulp_max / 2, math.inf),              # FLT_MAX + half an ulp: the tie rounds to 2^128
        (F32_MAX + ulp_max / 2 - 2.0 ** 76, F32_MAX),   # just below it
        (-(F32_MAX + ulp_max / 2), -math.inf),
        (2.0 ** -150, 0.0),                             # half the smallest subnormal: a tie to even zero
        (-(2.0 ** -150), -0.0),                         # underflow keeps the sign
        (2.0 ** -150 + 2.0 ** -170, 2.0 ** -149),
        (3 * 2.0 ** -150, 2.0 ** -148),                 # 1.5 subnormal ulps: a tie, to 2
        (5 * 2.0 ** -150, 2.0 ** -148),                 # 2.5 ulps: a tie, to 2
        (2.0 ** -126 - 2.0 ** -150, 2.0 ** -126),       # the largest subnormal + half an ulp rounds to the smallest normal
        (-0.0, -0.0), (0.0, 0.0),
    ]
    for x, want in cases:
        got = ew.f64_to_f32(x)
        assert er.same_value(got, want), (x, got, want)
        assert er.same_value(got, float(np.float64(x).astype(np.float32))), x


def test_f64_to_f32_matches_ieee_conversion_on_random_bits():
    rng = np.random.default_rng(11)
    b = rng.integers(0, 1 << 64, 4000, dtype=np.uint64, endpoint=False)
    # exponents near the float32 range too: subnormal, normal and overflowing results
    b[:2000] = (b[:2000] & np.uint64(0x800FFFFFFFFFFFFF)) | (rng.integers(1023 - 160, 1023 + 130, 2000).astype(np.uint64) << np.uint64(52))
    x = b.view(np.float64)
    want = x.astype(np.float32)
    got = np.array([ew.f64_to_f32(v) for v in x.tolist()], np.float64).astype(np.float32)
    er.assert_same(pa.array(got), pa.array(want), msg="f64 -> f32")


def test_int_to_float_double_rounding_traps():
    traps = {
        # value: the correctly rounded float32 (going through a double gives something else)
        2 ** 60 + 2 ** 36 + 1: 2.0 ** 60 + 2 ** 37,
        2 ** 63 + 2 ** 39 + 1: 2.0 ** 63 + 2 ** 40,     # uint64 at or above 2^63
        2 ** 64 - 1: 2.0 ** 64,
        -(2 ** 60 + 2 ** 36 + 1): -(2.0 ** 60 + 2 ** 37),
        2 ** 24 + 1: 2.0 ** 24, 2 ** 24 + 3: 2.0 ** 24 + 4,
    }
    for v, want in traps.items():
        assert ew.int_to_float(v, 32) == want, v
        t = pa.uint64() if v >= 2 ** 63 else pa.int64()
        got = pc.cast(pa.array([v], t), pa.float32(), safe=False)[0].as_py()
        assert got == want, f"reference {v}: {got} != {want}"
        if abs(v) > 2 ** 53 and v != 2 ** 64 - 1:   # the trap is real: through a double the value rounds twice
            assert float(np.float32(float(v))) != want, v
    assert ew.int_to_float(2 ** 53 + 1, 64) == 2.0 ** 53 and ew.int_to_float(2 ** 53 + 3, 64) == 2.0 ** 53 + 4


def test_integer_op_rules():
    i8, u8, i64 = pa.int8(), pa.uint8(), pa.int64()
    assert ew.int_op("divide", -7, 2, i8) == (-3, None)
    assert ew.int_op("divide", 7, -2, i8) == (-3, None)
    assert ew.int_op("divide", -128, -1, i8) == (0, None)
    assert ew.int_op("divide_checked", -128, -1, i8)[1] == "overflow"
    assert ew.int_op("divide", 5, 0, u8)[1] == "divide by zero"
    assert ew.int_op("add", 127, 1, i8) == (-128, None)
    assert ew.int_op("subtract_checked", 0, 1, u8)[1] == "overflow"
    assert ew.int_op("multiply", 2 ** 32, 2 ** 32, i64) == (0, None)
    assert ew.int_op("multiply_checked", -(2 ** 32), 2 ** 31, i64) == (-(2 ** 63), None)
    assert ew.int_op("multiply_checked", 2 ** 32, 2 ** 31, i64)[1] == "overflow"


def test_f64_exact_matches_ieee_double_on_random_operands():
    """the Fraction reference and the double unit agree on the four operations (both are correctly rounded)"""
    rng = np.random.default_rng(12)
    b = rng.integers(0, 1 << 64, (2, 600), dtype=np.uint64)
    b[:, :300] = (b[:, :300] & np.uint64(0x800FFFFFFFFFFFFF)) | (rng.integers(0, 60, (2, 300)).astype(np.uint64) << np.uint64(52))
    b[:, 300:400] = (b[:, 300:400] & np.uint64(0x800FFFFFFFFFFFFF)) | (rng.integers(2000, 2047, (2, 100)).astype(np.uint64) << np.uint64(52))
    x, y = b.view(np.float64)
    for base, f in (("add", np.add), ("subtract", np.subtract), ("multiply", np.multiply), ("divide", np.divide)):
        with np.errstate(all="ignore"):
            want = f(x, y)
        got = np.array([ew._f64_exact(base, a, c) for a, c in zip(x.tolist(), y.tolist())])
        er.assert_same(pa.array(got), pa.array(want), msg=base)
    assert math.copysign(1, ew._f64_exact("add", -0.0, -0.0)) < 0
    assert math.copysign(1, ew._f64_exact("add", 0.0, -0.0)) > 0
    assert math.copysign(1, ew._f64_exact("subtract", 1.0, 1.0)) > 0
    assert math.copysign(1, ew._f64_exact("multiply", -(2.0 ** -1000), 2.0 ** -1000)) < 0   # underflow keeps the sign


def test_float_to_int_restatement_matches_reference_scalar_path():
    """one element at a time the reference runs its scalar loop: there the convert() restatement must agree with it on
    NaN, +-inf and out-of-range values, for all twenty float -> int pairs"""
    for src in ew.FLOAT_TYPES:
        vals = [v for v in float_edges(src)] + [5e9, -5e9, 3e9, 2.0 ** 63, -(2.0 ** 63), 2.0 ** 64, 1.8e19, -1.5, 300.7, -129.5,
                                                65536.0, 2147483648.0, -2147483649.0]
        vals = [v if src == pa.float64() else float(np.float32(v)) for v in vals]
        for dst in ew.INT_TYPES:
            for v in vals:
                x = ew.to_array([v], src)
                want = pc.cast(x, dst, safe=False)[0].as_py()
                assert ew.float_to_int_unsafe(float(er.raw(x)[0]), dst) == want, (src, dst, v)


def test_float_to_uint32_depends_on_position_in_the_reference():
    """the reference's own unsafe float -> uint32 answer for an out-of-range value depends on where it sits (its vectorised
    loop body and its scalar tail disagree), so the device follows the documented convert() rule -- the scalar path -- and
    must not be "fixed" to match either position"""
    for src in ew.FLOAT_TYPES:
        answers = {n: pc.cast(pa.array([5e9] * n, src), pa.uint32(), safe=False)[-1].as_py() for n in (1, 7, 8, 9, 16, 17)}
        assert answers[1] == ew.float_to_int_unsafe(5e9, pa.uint32()) == 5_000_000_000 % (1 << 32)
        assert len(set(answers.values())) > 1, f"{src}: the reference no longer disagrees with itself: {answers}"
        nans = {n: pc.cast(pa.array([math.nan] * n, src), pa.uint32(), safe=False)[-1].as_py() for n in (1, 8)}
        assert nans[1] == ew.float_to_int_unsafe(math.nan, pa.uint32()) == 0


# ---------------------------------------------------------------------------------------------------------------------
# cast, arithmetic, compare, if_else: exact reference and oracle against pyarrow
# ---------------------------------------------------------------------------------------------------------------------
def in_range_for_unsafe(x: pa.Array, dst):
    """rows whose unsafe float -> int answer the reference defines (finite and in range after truncation)"""
    lo, hi = ew.int_range(dst)
    return [math.isfinite(v) and lo <= math.trunc(v) <= hi and not (dst.bit_width == 64 and abs(math.trunc(v)) >= 2 ** 63 and
                                                                      math.trunc(v) != lo) for v in ew.pylist(x)]


@pytest.mark.parametrize("src", ew.NUMERIC, ids=str)
def test_cast_vs_pyarrow(src):
    vals = edges(src) + ([2 ** 53 + 1, -(2 ** 24) - 1, 2 ** 24 + 1] if src in (pa.int64(),) else [])
    if src == pa.uint64():
        vals += [2 ** 63 + 2 ** 39 + 1, 2 ** 53 + 1]
    if pa.types.is_floating(src):
        vals += [1.5, -2.5, 127.9, -128.9, 255.5, 1e10, -1e10, 2.0 ** 31, 2.0 ** 63, 2.0 ** 64]
        vals = [v if src == pa.float64() else float(np.float32(v)) for v in vals]
    n = len(vals)
    x = ew.to_array(vals, src, np.arange(n) % 6 != 5)
    for dst in ew.NUMERIC:
        if dst == src:
            continue
        for safe in (True, False):
            msg = f"cast {src} -> {dst} safe={safe}"
            want = outcome(lambda: pc.cast(x, dst, safe=safe))
            if not safe and pa.types.is_floating(src) and pa.types.is_integer(dst):
                keep = pa.array(in_range_for_unsafe(x, dst))   # out-of-range answers: see the restatement tests
                got = ew.cast(x, dst, safe=False)
                er.assert_same(got.filter(keep), want[1].filter(keep), msg=msg)
                er.assert_same(ora.cast_array(x, dst, safe=False).filter(keep), want[1].filter(keep), msg="oracle " + msg)
                continue
            same_outcome(outcome(lambda: ew.cast(x, dst, safe=safe)), want, msg)
            same_outcome(outcome(lambda: ora.cast_array(x, dst, safe=safe)), want, "oracle " + msg)
            # every single offending value on its own, to pin the error text of each
            if safe and want[0] != "ok":
                for i in range(n):
                    one = x.slice(i, 1)
                    same_outcome(outcome(lambda: ew.cast(one, dst, True)), outcome(lambda: pc.cast(one, dst, safe=True)),
                                 f"{msg} row {i}")


@pytest.mark.parametrize("tl", ew.NUMERIC, ids=str)
@pytest.mark.parametrize("data", ["edges", "tame"])
def test_arithmetic_vs_pyarrow(tl, data):
    for tr in ew.NUMERIC:
        vl, vr = (edges(tl), edges(tr)) if data == "edges" else (tame(tl), tame(tr))
        for shape in SHAPES:
            for left, right in operands(shape, tl, tr, vl, vr):
                for op in ew.ARITH_OPS:
                    msg = f"{op} {tl} {tr} {shape} {left if isinstance(left, pa.Scalar) else ''}{right if isinstance(right, pa.Scalar) else ''}"
                    want = outcome(lambda: pc.call_function(op, [left, right]))
                    same_outcome(outcome(lambda: ew.arithmetic(op, left, right)), want, msg)
                    if not (isinstance(left, pa.Scalar) and not left.is_valid or isinstance(right, pa.Scalar) and not right.is_valid):
                        same_outcome(outcome(lambda: ora.arithmetic(op, left, right)), want, "oracle " + msg)


def test_checked_error_names_the_last_offending_row():
    """the reference's status is overwritten by each failing row: the message is that of the last one"""
    a = pa.array([-128, 5, 9, 1], pa.int8())
    b = pa.array([-1, 0, 0, -1], pa.int8())
    for n_rows, want in ((2, "divide by zero"), (4, "divide by zero")):
        x, y = a.slice(0, n_rows), b.slice(0, n_rows)
        with pytest.raises(pa.ArrowInvalid, match=want):
            pc.divide_checked(x, y)
        with pytest.raises(pa.ArrowInvalid, match=want):
            ew.arithmetic("divide_checked", x, y)
        with pytest.raises(pa.ArrowInvalid, match=want):
            ora.arithmetic("divide_checked", x, y)
    x, y = pa.array([5, -128], pa.int8()), pa.array([0, -1], pa.int8())
    for fn in (pc.divide_checked, lambda p, q: ew.arithmetic("divide_checked", p, q), lambda p, q: ora.arithmetic("divide_checked", p, q)):
        with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
            fn(x, y)
    # a zero divisor under a null never raises
    masked = pa.array([1, 0], pa.int8(), mask=np.array([False, True]))
    for fn in (pc.divide, lambda p, q: ew.arithmetic("divide", p, q), lambda p, q: ora.arithmetic("divide", p, q)):
        assert fn(pa.array([4, 4], pa.int8()), masked).to_pylist() == [4, None]


@pytest.mark.parametrize("tl", ew.NUMERIC, ids=str)
def test_compare_vs_pyarrow(tl):
    for tr in ew.NUMERIC:
        for shape in SHAPES:
            for left, right in operands(shape, tl, tr, edges(tl), edges(tr)):
                for op in ew.COMPARE_OPS:
                    msg = f"{op} {tl} {tr} {shape}"
                    want = outcome(lambda: pc.call_function(op, [left, right]))
                    same_outcome(outcome(lambda: ew.compare(op, left, right)), want, msg)
                    if not (isinstance(left, pa.Scalar) and not left.is_valid or isinstance(right, pa.Scalar) and not right.is_valid):
                        same_outcome(outcome(lambda: ora.compare(op, left, right)), want, "oracle " + msg)


def test_compare_nan_scalar_and_signed_zeros():
    x = pa.array([math.nan, 0.0, -0.0, 1.0, -math.inf, None])
    for s in (pa.scalar(math.nan), pa.scalar(-0.0), pa.scalar(0.0), pa.scalar(math.nan, pa.float32())):
        for op in ew.COMPARE_OPS:
            for left, right in ((x, s), (s, x)):
                same_result(ew.compare(op, left, right), pc.call_function(op, [left, right]), msg=f"{op} {s}")
    assert ew.compare("equal", x, pa.scalar(-0.0)).to_pylist() == [False, True, True, False, False, None]


def bits_equal(got: pa.Array, want: pa.Array, msg=""):
    """if_else is a selection: validity equal and the value bits of every valid slot identical (NaN payloads, -0.0)"""
    assert got.type == want.type and len(got) == len(want), msg
    v = er.valid_mask(want)
    assert np.array_equal(er.valid_mask(got), v), msg
    gb, wb = er.bits(got)[v], er.bits(want)[v]
    bad = np.flatnonzero(gb != wb)
    assert not len(bad), f"{msg}: {len(bad)} differ, first at {np.flatnonzero(v)[bad[:3]]}: {gb[bad[:3]]} vs {wb[bad[:3]]}"


@pytest.mark.parametrize("tl", ew.NUMERIC, ids=str)
def test_if_else_vs_pyarrow(tl):
    for tr in ew.NUMERIC:
        a, b = pair_arrays(tl, tr, edges(tl), edges(tr))
        n = len(a)
        cond = pa.array(np.arange(n) % 3 != 1, mask=np.arange(n) % 11 == 10)
        for left, right in [(a, b)] + [(a, s) for s in scalars(tr)] + [(s, b) for s in scalars(tl)]:
            for c in (cond, pa.scalar(True), pa.scalar(False)):
                msg = f"if_else {tl} {tr} {left.type} {right.type}"
                want = outcome(lambda: pc.if_else(c, left, right))
                got = outcome(lambda: ew.if_else(c, left, right))
                assert got[0] == want[0], (msg, got, want)
                if got[0] != "ok":
                    assert got[1] == want[1], msg
                    assert outcome(lambda: ora.if_else(c, left, right)) == want, "oracle " + msg
                    continue
                (bits_equal if tl == tr else er.assert_same)(got[1], want[1], msg)
                null_scalar = any(isinstance(x, pa.Scalar) and not x.is_valid for x in (left, right))
                if not null_scalar:
                    (bits_equal if tl == tr else er.assert_same)(ora.if_else(c, left, right), want[1], "oracle " + msg)


# ---------------------------------------------------------------------------------------------------------------------
# the implicit safe cast of scalar operands
# ---------------------------------------------------------------------------------------------------------------------
IMPLICIT_CASES = [
    ("add", pa.array([1.0], pa.float32()), pa.scalar(2 ** 25 + 1)),
    ("less", pa.array([1.0], pa.float32()), pa.scalar(2 ** 25 + 1)),
    ("if_else", pa.array([1.0], pa.float32()), pa.scalar(2 ** 25 + 1)),
    ("add", pa.array([1.0], pa.float64()), pa.scalar(2 ** 53 + 1)),
    ("less", pa.array([1.0], pa.float64()), pa.scalar(2 ** 53 + 1)),
    ("if_else", pa.array([1.0], pa.float64()), pa.scalar(2 ** 53 + 1)),
    ("less", pa.array([1], pa.int8()), pa.scalar(2 ** 64 - 1, pa.uint64())),
    ("add", pa.array([1], pa.int32()), pa.scalar(2 ** 63, pa.uint64())),
    ("add", pa.array([1.0], pa.float32()), pa.scalar(2 ** 25 + 1, pa.uint32())),
    ("if_else", pa.array([2 ** 25 + 1], pa.int64()), pa.array([1.0], pa.float32())),
    ("if_else", pa.array([1.0], pa.float32()), pa.array([2 ** 25 + 1], pa.int64())),
]


def _call(impl, fn, left, right):
    if fn == "if_else":
        return impl.if_else(pa.array([True]), left, right)
    return (pc.call_function(fn, [left, right]) if impl is pc else
            (impl.arithmetic if fn == "add" else impl.compare)(fn, left, right))


@pytest.mark.parametrize("case", range(len(IMPLICIT_CASES)))
def test_implicit_cast_raises_like_the_reference(case):
    fn, left, right = IMPLICIT_CASES[case]
    want = outcome(lambda: _call(pc, fn, left, right))
    assert want[0] == "ArrowInvalid", want
    for a, b in ((left, right), (right, left) if isinstance(right, pa.Array) or fn != "if_else" else (left, right)):
        if not isinstance(a, pa.Array) and not isinstance(b, pa.Array):
            continue
        assert outcome(lambda: _call(ew, fn, a, b))[1] == outcome(lambda: _call(pc, fn, a, b))[1]
        assert outcome(lambda: _call(ora, fn, a, b)) == outcome(lambda: _call(pc, fn, a, b)), (fn, a, b)


def scalar_bits_or_error(s: pa.Scalar, dst: pa.DataType):
    """what the reference's safe cast makes of the scalar: the value bits of the result, or the error text"""
    kind, r = outcome(lambda: pc.cast(pa.array([s], s.type), dst, safe=True))
    if kind != "ok":
        return kind, r
    return "ok", int(er.bits(r)[0])


@pytest.mark.parametrize("src", ew.NUMERIC, ids=str)
def test_scalar_to_is_the_reference_safe_cast(src):
    """compute._scalar_to (host-side argument preparation for the device kernels) against the reference's safe cast, for
    every target CommonNumeric can pick; a scalar of the target type keeps its exact bits"""
    vals = edges(src)
    if src in (pa.int64(), pa.uint64(), pa.int32(), pa.uint32()):
        vals += [v for v in (2 ** 24, 2 ** 24 + 1, -(2 ** 24), -(2 ** 24) - 1, 2 ** 53, 2 ** 53 + 1, -(2 ** 53) - 1, 2 ** 63 + 1)
                 if ew.int_range(src)[0] <= v <= ew.int_range(src)[1]]
    if src == pa.float32():
        vals.append(f32_bits(0x7F800001))                           # a signalling NaN
    for dst in ew.NUMERIC:
        if ew.common_numeric([src, dst]) != dst:
            continue                                                # never dispatched
        for v in vals:
            s = ew.to_array([v], src)[0] if not (src == pa.float32() and math.isnan(v)) else \
                pa.array(np.array([0x7F800001], np.uint32).view(np.float32))[0]
            want = scalar_bits_or_error(s, dst)
            got = outcome(lambda: bc._scalar_to(s, type_id(dst)))
            assert got[0] == want[0], (src, dst, v, got, want)
            if got[0] == "ok":
                mask = (1 << dst.bit_width) - 1
                if pa.types.is_floating(dst) and src != dst and math.isnan(v):
                    continue                                        # a converted NaN: any payload
                assert got[1].bits & mask == want[1], (src, dst, v, hex(got[1].bits), hex(want[1]))
            else:
                assert got[1] == want[1], (src, dst, v)
