"""The device's numeric math functions against tests/math_ref.py: every function over every type it takes, lengths
around the applicator's tiles, unaligned offsets, array / scalar / null-scalar operands, every error path with its
text, launches per call, both options forms of call_function, and 2^26-row checks of abs, sqrt, round, bit_wise_and,
shift_right and round_to_multiple."""
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import math_ref as mr
from tests.test_math_oracle import PA_TYPE, edges, same, to_py

pytestmark = pytest.mark.gpu

# map1 / map2 tiles: 32 lanes x V x 4 accesses per warp, 8 warps per block
WARP_TILE = {1: 32 * 16 * 4, 2: 32 * 8 * 4, 4: 32 * 4 * 4, 8: 32 * 2 * 4}
OFFSETS = [0, 1, 3, 7, 63]
ERRORS = {"Invalid": pa.ArrowInvalid, "NotImplemented": pa.ArrowNotImplementedError}


def width(t):
    return 4 if t == "float" else 8 if t == "double" else mr.bits(t) // 8


def column(t, n, offset, seed, nulls=True):
    """a pyarrow array of n values of type t sliced at `offset`, drawn from the edge values, about 10 % null"""
    rng = np.random.default_rng(seed)
    pool = edges(t)
    vals = [pool[i] for i in rng.integers(0, len(pool), n + offset)]
    mask = rng.random(n + offset) < 0.1 if nulls else None
    return pa.array(vals, PA_TYPE[t], mask=mask).slice(offset)


def lengths(t):
    w = WARP_TILE[width(t)]
    return [0, 1, w - 1, w, w + 1, 8 * w - 1, 8 * w + 1]


def expect(ref_fn, dev_fn, t):
    try:
        want = ("ok", ref_fn())
    except mr.MathError as e:
        want = (e.kind, e.message)
    if want[0] == "ok":
        got = dev_fn().to_arrow().to_pylist()
        same(got, to_py(want[1], t), t)
    else:
        with pytest.raises(ERRORS[want[0]]) as ei:
            dev_fn()
        if want[0] == "Invalid":
            assert str(ei.value) == want[1] or want[1] in str(ei.value)


def launches(fn):
    before = _cabi.lib().b2_launch_count()
    fn()
    return _cabi.lib().b2_launch_count() - before


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", mr.INT_TYPES + mr.FLOAT_TYPES)
@pytest.mark.parametrize("name", mr.UNARY)
def test_unary(ctx, name, t):
    for n in lengths(t)[:4]:
        for off in OFFSETS:
            a = column(t, n, off, n * 7 + off)
            d = DeviceArray.from_arrow(a, ctx)
            expect(lambda: mr.unary(name, a.to_pylist(), t)[0], lambda: getattr(bc, name)(d), mr.unary_out_type(name, t))


def test_unary_errors_and_launches(ctx):
    d = DeviceArray.from_arrow(pa.array([-128, 5, None], pa.int8()), ctx)
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.abs_checked(d)
    with pytest.raises(pa.ArrowNotImplementedError, match="negate_checked"):
        bc.negate_checked(DeviceArray.from_arrow(pa.array([1], pa.uint8()), ctx))
    with pytest.raises(pa.ArrowInvalid, match="square root of negative number"):
        bc.sqrt_checked(DeviceArray.from_arrow(pa.array([4.0, -1.0]), ctx))
    # a failing value under a null is not checked
    masked = DeviceArray.from_arrow(pa.array([-128, 5], pa.int8(), mask=np.array([True, False])), ctx)
    assert bc.abs_checked(masked).to_arrow().to_pylist() == [None, 5]
    no_nulls = DeviceArray.from_arrow(pa.array([1.5, -2.5] * 1000), ctx)
    with_nulls = DeviceArray.from_arrow(pa.array([1.5, None, -2.5] * 1000).slice(3), ctx)
    assert launches(lambda: bc.abs(no_nulls)) == 1
    assert launches(lambda: bc.abs(with_nulls)) == 2


def test_sign_bits(ctx):
    d = DeviceArray.from_arrow(pa.array([-0.0, float("nan"), 0.0, -3.0, float("-inf")]), ctx)
    got = bc.sign(d).to_arrow()
    raw = np.frombuffer(got.buffers()[1], np.float64)[: len(got)]
    assert raw[0].tobytes() == np.float64(0.0).tobytes() and np.isnan(raw[1]) and list(raw[2:]) == [0.0, -1.0, -1.0]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", mr.INT_TYPES)
@pytest.mark.parametrize("name", mr.BINARY)
def test_binary(ctx, name, t):
    rng = np.random.default_rng(zlib.crc32(f"{name}-{t}".encode()))
    for n in lengths(t)[:4]:
        for off in (0, 3, 63):
            a = column(t, n, off, n + off)
            if name.startswith("shift"):
                pool = list(range(-1, mr.bits(t) + 2))
            elif name.startswith("power"):
                pool = list(range(0, 65))
            else:
                pool = edges(t)
            lo, hi = mr.lo_hi(t)
            pool = [v for v in pool if lo <= v <= hi]
            b = pa.array([pool[i] for i in rng.integers(0, len(pool), n + off)], PA_TYPE[t],
                         mask=rng.random(n + off) < 0.1).slice(off)
            da, db = DeviceArray.from_arrow(a, ctx), DeviceArray.from_arrow(b, ctx)
            expect(lambda: mr.binary(name, a.to_pylist(), b.to_pylist(), t), lambda: getattr(bc, name)(da, db), t)
            s = pool[len(pool) // 2]
            expect(lambda: mr.binary(name, a.to_pylist(), s, t),
                   lambda: getattr(bc, name)(da, pa.scalar(s, PA_TYPE[t])), t)
            expect(lambda: mr.binary(name, s, b.to_pylist(), t),
                   lambda: getattr(bc, name)(pa.scalar(s, PA_TYPE[t]), db), t)
            expect(lambda: mr.binary(name, a.to_pylist(), None, t),
                   lambda: getattr(bc, name)(da, pa.scalar(None, PA_TYPE[t])), t)


def test_binary_errors(ctx):
    i8 = lambda v, m=None: DeviceArray.from_arrow(pa.array(v, pa.int8(), mask=m), ctx)  # noqa: E731
    # unchecked power checks the slot under a null; power_checked does not
    exps = pa.Array.from_buffers(pa.int8(), 2, [pa.py_buffer(bytes([0b01])), pa.py_buffer(np.array([2, -1], np.int8).tobytes())])
    dexps = DeviceArray.from_arrow(exps, ctx)
    with pytest.raises(pa.ArrowInvalid, match=mr.NEGATIVE_POWER):
        bc.power(i8([3, 3]), dexps)
    assert bc.power_checked(i8([3, 3]), dexps).to_arrow().to_pylist() == [9, None]
    assert bc.power(i8([2]), i8([7])).to_arrow().to_pylist() == [-128]
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.power_checked(i8([2]), i8([7]))
    # the last failing row names the message
    with pytest.raises(pa.ArrowInvalid, match=mr.NEGATIVE_POWER):
        bc.power_checked(i8([2, 2]), i8([7, -1]))
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.power_checked(i8([2, 2]), i8([-1, 7]))
    assert bc.shift_left_checked(i8([64]), i8([1])).to_arrow().to_pylist() == [-128]
    with pytest.raises(pa.ArrowInvalid, match="shift amount must be >= 0"):
        bc.shift_left_checked(i8([1]), i8([7]))
    with pytest.raises(pa.ArrowNotImplementedError, match="no kernel matching"):
        bc.power(DeviceArray.from_arrow(pa.array([2.0]), ctx), 2.0)
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.bit_wise_and(DeviceArray.from_arrow(pa.array([2.0]), ctx), 1)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", mr.INT_TYPES + mr.FLOAT_TYPES)
@pytest.mark.parametrize("mode", mr.ROUND_MODES)
def test_round(ctx, mode, t):
    digits = [-400, -309, -20, -3, -2, -1, 0, 1, 2, 11, 20, 308, 400] if t in mr.FLOAT_TYPES else \
        list(range(-(mr.DIGITS10[t] + 1), 2))
    for n, off in ((lengths(t)[2], 1), (lengths(t)[3], 0), (lengths(t)[4], 7)):
        a = column(t, n, off, n + off)
        d = DeviceArray.from_arrow(a, ctx)
        vals = a.to_pylist()
        for nd in digits:
            if t == "uint64" and nd == -19:
                continue
            expect(lambda: mr.round_(vals, t, nd, mode), lambda: bc.round(d, nd, mode), t)
        mults = ([1.5, 0.25, 1e-30, 1e30] if t == "float" else [1.5, 0.25, 1e-300, 1e300]) if t in mr.FLOAT_TYPES else [1, 3, 10, 1000 if mr.bits(t) > 8 else 100,
                                                                         mr.lo_hi(t)[1]]
        for m in mults:
            mm = np.float32(m) if t == "float" else m
            expect(lambda: mr.round_to_multiple(vals, t, mm, mode),
                   lambda: bc.round_to_multiple(d, pa.scalar(m, PA_TYPE[t]), mode), t)
        rng = np.random.default_rng(n)
        ds = pa.array(rng.integers(-22, 5, len(vals)).astype(np.int32), mask=rng.random(len(vals)) < 0.1)
        dd = DeviceArray.from_arrow(ds, ctx)
        expect(lambda: mr.round_binary(vals, t, ds.to_pylist(), mode), lambda: bc.round_binary(d, dd, mode), t)
        expect(lambda: mr.round_binary(vals, t, -1, mode), lambda: bc.round_binary(d, pa.scalar(-1, pa.int32()), mode), t)
        expect(lambda: mr.round_binary(vals, t, None, mode),
               lambda: bc.round_binary(d, pa.scalar(None, pa.int32()), mode), t)


def test_round_pins(ctx):
    d = DeviceArray.from_arrow(pa.array([0.7]), ctx)
    assert bc.round(d, 11).to_arrow().to_pylist() == [0.699999999996]
    with pytest.raises(pa.ArrowInvalid, match="overflow occurred during rounding"):
        bc.round(DeviceArray.from_arrow(pa.array([1.5]), ctx), 400)
    i8 = DeviceArray.from_arrow(pa.array([1, 125], pa.int8()), ctx)
    with pytest.raises(pa.ArrowInvalid, match="Rounding to -3 digits is out of range for type int8"):
        bc.round(i8, -3)
    with pytest.raises(pa.ArrowInvalid, match="Integer value 1000 not in range: -128 to 127"):
        bc.round_to_multiple(i8, 1000)
    with pytest.raises(pa.ArrowInvalid, match="Rounding multiple must be positive"):
        bc.round_to_multiple(i8, 0)
    with pytest.raises(pa.ArrowInvalid, match="Rounding multiple must be non-null and valid"):
        bc.round_to_multiple(i8, pa.scalar(None, pa.int8()))
    # int8 values are printed as numbers (pyarrow prints them as characters)
    with pytest.raises(pa.ArrowInvalid, match="^Rounding 125 up to multiple of 10 would overflow$"):
        bc.round_to_multiple(i8, 10, "up")
    i32 = DeviceArray.from_arrow(pa.array([2 ** 31 - 1, 5, 2 ** 31 - 2], pa.int32()), ctx)
    with pytest.raises(pa.ArrowInvalid, match="^Rounding 2147483646 up to multiples of 1073741825 would overflow$"):
        bc.round_to_multiple(i32, 2 ** 30 + 1)
    # float32: round scales in float32, round_binary in float64
    from tests.test_math_oracle import float32_round_grid
    grid = [v for v, nd in float32_round_grid() if nd == 2]
    f = DeviceArray.from_arrow(pa.array(grid, pa.float32()), ctx)
    same(bc.round(f, 2).to_arrow().to_pylist(), to_py(mr.round_(grid, "float", 2), "float"), "float")
    same(bc.round_binary(f, 2).to_arrow().to_pylist(), to_py(mr.round_binary(grid, "float", [2] * len(grid)), "float"),
         "float")
    assert bc.round(f, 2).to_arrow() != bc.round_binary(f, 2).to_arrow()


def test_round_launches(ctx):
    d = DeviceArray.from_arrow(pa.array(np.arange(5000, dtype=np.int64)), ctx)
    assert launches(lambda: bc.round_to_multiple(d, 10)) == 1
    assert launches(lambda: bc.round(d, -2)) == 1
    assert launches(lambda: bc.round(d, 2)) == 0  # the identity: one copy
    dn = DeviceArray.from_arrow(pa.array(np.arange(5003, dtype=np.float64), mask=np.arange(5003) % 3 == 0).slice(3), ctx)
    assert launches(lambda: bc.round(dn, 2)) == 2


def test_call_function_options(ctx):
    d = DeviceArray.from_arrow(pa.array([1.25, -2.35, 1234.5, None]), ctx)
    i = DeviceArray.from_arrow(pa.array([125, -175, None], pa.int64()), ctx)
    s = DeviceArray.from_arrow(pa.array([1, 0, -1, 2], pa.int32()), ctx)
    cases = [
        ("round", [d], pc.RoundOptions(1, "half_up"), {"ndigits": 1, "round_mode": "half_up"}, bc.round(d, 1, "half_up")),
        ("round_to_multiple", [i], pc.RoundToMultipleOptions(pa.scalar(50, pa.int64()), "down"),
         {"multiple": 50, "round_mode": "down"}, bc.round_to_multiple(i, 50, "down")),
        ("round_to_multiple", [d], pc.RoundToMultipleOptions(0.5, "up"), {"multiple": 0.5, "round_mode": "up"},
         bc.round_to_multiple(d, 0.5, "up")),
        ("round_binary", [d, s], pc.RoundBinaryOptions("towards_zero"), {"round_mode": "towards_zero"},
         bc.round_binary(d, s, "towards_zero")),
    ]
    for name, args, obj, kw, want in cases:
        assert name in bc.list_functions()
        assert bc.call_function(name, args, obj).to_arrow().equals(want.to_arrow()), name
        assert bc.call_function(name, args, kw).to_arrow().equals(want.to_arrow()), name
    assert bc.call_function("abs", [d]).to_arrow().equals(bc.abs(d).to_arrow())


# ---------------------------------------------------------------------------------------------------------------------
N_BIG = 1 << 26


def test_large(ctx):
    """2^26 rows per family against vectorised numpy restatements (each numpy op is one IEEE operation)"""
    rng = np.random.default_rng(5)
    x = (rng.random(N_BIG) - 0.5) * 2e6
    arr = DeviceArray.from_arrow(pa.array(x), ctx)
    got = lambda d: d.to_arrow().to_numpy(zero_copy_only=False)  # noqa: E731
    assert np.array_equal(got(bc.abs(arr)).view(np.uint64), np.abs(x).view(np.uint64))
    assert np.array_equal(got(bc.sqrt(bc.abs(arr))), np.sqrt(np.abs(x)))
    # round(x, 2), half_to_even
    r = x * 100.0
    frac = r - np.floor(r)
    t = np.trunc(r)
    nearest = np.where(np.abs(r - t) >= 0.5, t + np.sign(r), t)
    half = r * 0.5
    th = np.trunc(half)
    tie = (th + np.where(np.abs(half - th) >= 0.5, np.sign(half), 0.0)) * 2.0
    want = np.where(frac == 0, x, np.where(frac != 0.5, nearest, tie) / 100.0)
    assert np.array_equal(got(bc.round(arr, 2)).view(np.uint64), want.view(np.uint64))
    del x, r, frac, t, nearest, half, th, tie, want, arr
    xi = rng.integers(-(1 << 62), 1 << 62, N_BIG, dtype=np.int64)
    ai = DeviceArray.from_arrow(pa.array(xi), ctx)
    assert np.array_equal(got(bc.bit_wise_and(ai, pa.scalar(0xFFFF, pa.int64()))), xi & 0xFFFF)
    assert np.array_equal(got(bc.shift_right(ai, pa.scalar(4, pa.int64()))), xi >> 4)
    q = np.sign(xi) * (np.abs(xi) // 1000) * 1000
    rem = np.abs(xi - q)
    up = np.where(xi >= 0, q + 1000, q - 1000)
    odd = (q // 1000) % 2 != 0
    want_i = np.where(rem * 2 > 1000, up, np.where((rem * 2 == 1000) & odd, up, q))
    assert np.array_equal(got(bc.round_to_multiple(ai, 1000)), want_i)
