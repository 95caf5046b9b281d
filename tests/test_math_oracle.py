"""tests/math_ref.py against the reference's own expected cases (tests/golden/kat_math.json) and against
pyarrow.compute, for every function over every type it takes."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import math_ref as mr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_math.json")
PA_TYPE = {t: getattr(pa, t if t not in ("float", "double") else {"float": "float32", "double": "float64"}[t])()
           for t in mr.INT_TYPES + mr.FLOAT_TYPES}

F64_EDGES = [0.0, -0.0, 0.5, -0.5, 1.5, 2.5, -2.5, 0.7, 1.005, 2.675, 123.456, -123.456, 1e-300, 5e-324, -5e-324,
             1e300, 1.7976931348623157e308, -1.7976931348623157e308, float("inf"), float("-inf"), float("nan"),
             np.nextafter(0.5, 1), np.nextafter(0.5, 0), np.nextafter(2.5, 3), np.nextafter(2.5, 2), 1234.5, -1234.5,
             4503599627370496.5 - 0.5, 0.125, 0.375, 9.995, -9.995]
F32_EDGES = [float(np.float32(v)) for v in F64_EDGES if not (abs(v) > 3.4e38 and np.isfinite(v)) and abs(v) >= 1e-38
             or v == 0] + [3.4028234663852886e38, -3.4028234663852886e38, 1e-45, float(np.nextafter(np.float32(0.5),
                                                                                                    np.float32(1)))]


def edges(t):
    if t == "double":
        return list(F64_EDGES)
    if t == "float":
        return list(F32_EDGES)
    lo, hi = mr.lo_hi(t)
    vals = {lo, lo + 1, hi, hi - 1, 0, 1, 2, 3, 5, 7, 10, 15, 25, 45, 99, 100, 125, 127, 150, 250}
    if mr.signed(t):
        vals |= {-1, -2, -3, -5, -7, -10, -15, -25, -45, -99, -100, -125, -127, -150, -250}
    for k in range(1, mr.DIGITS10[t] + 1):
        vals |= {10 ** k, 10 ** k // 2, 10 ** k // 2 + 1, 3 * 10 ** k + 10 ** k // 2}
        if mr.signed(t):
            vals |= {-(10 ** k // 2), -(3 * 10 ** k + 10 ** k // 2)}
    return sorted(v for v in vals if lo <= v <= hi)


def to_py(values, t):
    return [None if v is None else (float(v) if t in mr.FLOAT_TYPES else int(v)) for v in values]


def same(got, want, t):
    """float lists bit for bit (any NaN matches any NaN: payloads differ by platform); others exactly"""
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if g is None or w is None:
            assert g is None and w is None
        elif t in mr.FLOAT_TYPES or isinstance(w, float):
            f = np.float32 if t == "float" else np.float64
            if np.isnan(w):
                assert np.isnan(g)
            else:
                assert np.array([g], f).tobytes() == np.array([w], f).tobytes(), (g, w)
        else:
            assert int(g) == int(w)


def run_ref(fn):
    try:
        return "ok", fn()
    except mr.MathError as e:
        return e.kind, e.message


def run_pa(fn):
    try:
        return "ok", fn()
    except pa.ArrowNotImplementedError as e:
        return "NotImplemented", str(e)
    except pa.ArrowInvalid as e:
        return "Invalid", str(e)


def check(ref, got, t, text=True):
    assert ref[0] == got[0], (ref, got)
    if ref[0] == "ok":
        same(to_py(ref[1], t), got[1].to_pylist(), t)
    elif text and ref[0] == "Invalid":
        assert ref[1] == got[1]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", mr.INT_TYPES + mr.FLOAT_TYPES)
@pytest.mark.parametrize("name", mr.UNARY)
def test_unary_against_pyarrow(name, t):
    vals = edges(t) + [None]
    ref = run_ref(lambda: mr.unary(name, vals, t)[0])
    got = run_pa(lambda: getattr(pc, name)(pa.array(vals, PA_TYPE[t])))
    out_t = mr.unary_out_type(name, t)
    check(ref, got, out_t)
    if ref[0] == "ok":
        assert str(got[1].type) == str(PA_TYPE[out_t])


def test_sign_of_zero_and_nan_bits():
    got, _ = mr.unary("sign", [np.float64(-0.0), np.float64(np.nan)], "double")
    assert np.array(got[:1]).tobytes() == np.array([0.0]).tobytes()
    assert np.isnan(got[1])


@pytest.mark.parametrize("t", mr.INT_TYPES)
@pytest.mark.parametrize("name", mr.BINARY)
def test_binary_against_pyarrow(name, t):
    lo, hi = mr.lo_hi(t)
    if name.startswith("shift"):
        amounts = list(range(-1, mr.bits(t) + 2))
    elif name.startswith("power"):
        amounts = list(range(0, 65)) + [-1, -2]
    else:
        amounts = edges(t)
    amounts = [a for a in amounts if lo <= a <= hi]
    bases = [v for v in edges(t) if abs(v) < 300 or v in (lo, hi)][:24]
    pairs = [(b, a) for b in bases for a in amounts]
    pairs = [p for p in pairs if not name.startswith("power") or p[1] >= 0]
    left, right = [p[0] for p in pairs], [p[1] for p in pairs]
    ref = run_ref(lambda: mr.binary(name, left, right, t))
    got = run_pa(lambda: getattr(pc, name)(pa.array(left, PA_TYPE[t]), pa.array(right, PA_TYPE[t])))
    check(ref, got, t)
    # one row at a time for the errors: the message of each failing row
    for l, r in pairs[:: max(1, len(pairs) // 200)]:
        check(run_ref(lambda: mr.binary(name, [l], [r], t)),
              run_pa(lambda: getattr(pc, name)(pa.array([l], PA_TYPE[t]), pa.array([r], PA_TYPE[t]))), t)


@pytest.mark.parametrize("name", ["power", "power_checked"])
def test_negative_exponent(name):
    for t in ("int8", "int64"):
        ref = run_ref(lambda: mr.binary(name, [2, 3], [1, -1], t))
        got = run_pa(lambda: getattr(pc, name)(pa.array([2, 3], PA_TYPE[t]), pa.array([1, -1], PA_TYPE[t])))
        check(ref, got, t)


def test_negative_exponent_under_a_null():
    """unchecked power checks every slot: a negative exponent under a null raises; power_checked does not look"""
    exps = pa.Array.from_buffers(pa.int8(), 2, [pa.py_buffer(bytes([0b01])), pa.py_buffer(np.array([2, -1], np.int8).tobytes())])
    base = pa.array([3, 3], pa.int8())
    with pytest.raises(pa.ArrowInvalid, match=mr.NEGATIVE_POWER):
        pc.power(base, exps)
    assert pc.power_checked(base, exps).to_pylist() == [9, None]
    with pytest.raises(mr.MathError, match=mr.NEGATIVE_POWER):
        mr.binary("power", [3, 3], [2, None], "int8", right_under_nulls=[2, -1])
    assert mr.binary("power_checked", [3, 3], [2, None], "int8", right_under_nulls=[2, -1]) == [9, None]


def test_null_scalars():
    for name in ("power", "bit_wise_and", "shift_left_checked"):
        assert mr.binary(name, [1, 2], None, "int32") == [None, None]
        assert getattr(pc, name)(pa.array([1, 2], pa.int32()), pa.scalar(None, pa.int32())).to_pylist() == [None, None]
    assert mr.round_binary([1.5, 2.5], "double", None) == [None, None]
    assert pc.round_binary(pa.array([1.5, 2.5]), pa.scalar(None, pa.int32())).to_pylist() == [None, None]


def test_last_failing_row_names_the_message():
    t = "int32"
    vals = [2 ** 31 - 1, 5, -(2 ** 31), 2 ** 31 - 2]
    for mode in ("up", "down", "half_up", "towards_infinity"):
        ref = run_ref(lambda: mr.round_to_multiple(vals, t, 10, mode))
        got = run_pa(lambda: pc.round_to_multiple(pa.array(vals, pa.int32()), multiple=10, round_mode=mode))
        check(ref, got, t)
    exps = [1, -1, 2, -2]
    check(run_ref(lambda: mr.binary("power", [2] * 4, exps, "int64")),
          run_pa(lambda: pc.power(pa.array([2] * 4, pa.int64()), pa.array(exps, pa.int64()))), "int64")


# ---------------------------------------------------------------------------------------------------------------------
NDIGITS = [-400, -309] + list(range(-20, 21)) + [38, 39, 308, 400]


@pytest.mark.parametrize("t", mr.FLOAT_TYPES)
@pytest.mark.parametrize("mode", mr.ROUND_MODES)
def test_round_float_against_pyarrow(mode, t):
    vals = edges(t) + [None]
    for nd in NDIGITS:
        ref = run_ref(lambda: mr.round_(vals, t, nd, mode))
        got = run_pa(lambda: pc.round(pa.array(vals, PA_TYPE[t]), ndigits=nd, round_mode=mode))
        check(ref, got, t)
        # each finite value alone, so that one failing row does not hide the others
        if ref[0] != "ok":
            for v in vals[::3]:
                check(run_ref(lambda: mr.round_([v], t, nd, mode)),
                      run_pa(lambda: pc.round(pa.array([v], PA_TYPE[t]), ndigits=nd, round_mode=mode)), t)


def test_round_uses_the_float_powers_of_ten():
    assert mr.round_([0.7], "double", 11) == [np.float64(0.699999999996)]
    assert pc.round(pa.array([0.7]), 11).to_pylist() == [0.699999999996]
    assert float(mr.pow10(11)) == 99999997952.0


@pytest.mark.parametrize("t", mr.FLOAT_TYPES)
@pytest.mark.parametrize("mode", mr.ROUND_MODES)
def test_round_binary_float_against_pyarrow(mode, t):
    vals = edges(t)
    for nd in [-400, -309, -20, -5, -1, 0, 1, 2, 5, 11, 20, 38, 39, 308, 400]:
        ref = run_ref(lambda: mr.round_binary(vals, t, [nd] * len(vals), mode))
        got = run_pa(lambda: pc.round_binary(pa.array(vals, PA_TYPE[t]), pa.array([nd] * len(vals), pa.int32()),
                                             round_mode=mode))
        check(ref, got, t)


def float32_round_grid():
    """float32 values where round (scaling in float32) and round_binary (scaling in float64) differ"""
    rng = np.random.default_rng(7)
    vals = rng.uniform(-1000, 1000, 4000).astype(np.float32)
    out = []
    for nd in (1, 2, 3, 4):
        a = mr.round_([float(v) for v in vals], "float", nd)
        b = mr.round_binary([float(v) for v in vals], "float", [nd] * len(vals))
        out += [(float(v), nd) for v, x, y in zip(vals, a, b) if np.float32(x) != np.float32(y)]
    return out


def test_float32_round_and_round_binary_differ_and_both_match():
    grid = float32_round_grid()
    assert len(grid) > 10
    for nd in (1, 2, 3, 4):
        vals = [v for v, d in grid if d == nd]
        if not vals:
            continue
        check(run_ref(lambda: mr.round_(vals, "float", nd)), run_pa(lambda: pc.round(pa.array(vals, pa.float32()), nd)),
              "float")
        check(run_ref(lambda: mr.round_binary(vals, "float", [nd] * len(vals))),
              run_pa(lambda: pc.round_binary(pa.array(vals, pa.float32()), pa.array([nd] * len(vals), pa.int32()))),
              "float")


@pytest.mark.parametrize("t", mr.INT_TYPES)
@pytest.mark.parametrize("mode", mr.ROUND_MODES)
def test_round_integer_against_pyarrow(mode, t):
    vals = edges(t)
    # int8 / uint8 overflow messages print the values as characters in pyarrow: match the error class only there
    text = mr.bits(t) > 8
    for nd in range(-(mr.DIGITS10[t] + 2), 3):
        if t == "uint64" and nd == -19:
            continue  # pyarrow 24 reads past its power-of-ten table here (10^19 is the device's and the restatement's)
        ref = run_ref(lambda: mr.round_(vals, t, nd, mode))
        got = run_pa(lambda: pc.round(pa.array(vals, PA_TYPE[t]), ndigits=nd, round_mode=mode))
        check(ref, got, t, text)
        if ref[0] == "Invalid":
            for v in vals:
                check(run_ref(lambda: mr.round_([v], t, nd, mode)),
                      run_pa(lambda: pc.round(pa.array([v], PA_TYPE[t]), ndigits=nd, round_mode=mode)), t, text)
    lo, hi = mr.lo_hi(t)
    for m in sorted({1, 2, 3, 7, hi, hi // 2, hi // 2 + 1} | {10 ** k for k in range(1, mr.DIGITS10[t] + 1)}):
        ref = run_ref(lambda: mr.round_to_multiple(vals, t, m, mode))
        got = run_pa(lambda: pc.round_to_multiple(pa.array(vals, PA_TYPE[t]), multiple=pa.scalar(m, PA_TYPE[t]),
                                                  round_mode=mode))
        check(ref, got, t, text)
        if ref[0] == "Invalid":
            for v in vals:
                check(run_ref(lambda: mr.round_to_multiple([v], t, m, mode)),
                      run_pa(lambda: pc.round_to_multiple(pa.array([v], PA_TYPE[t]), multiple=pa.scalar(m, PA_TYPE[t]),
                                                          round_mode=mode)), t, text)


@pytest.mark.parametrize("t", ["int8", "int32", "uint32", "int64", "uint64"])
def test_round_binary_integer_against_pyarrow(t):
    vals = edges(t)
    for mode in mr.ROUND_MODES:
        for nd in [-(mr.DIGITS10[t] + 1), -mr.DIGITS10[t] + (t == "uint64"), -3, -2, -1, 0, 4]:
            ref = run_ref(lambda: mr.round_binary(vals, t, [nd] * len(vals), mode))
            got = run_pa(lambda: pc.round_binary(pa.array(vals, PA_TYPE[t]), pa.array([nd] * len(vals), pa.int32()),
                                                 round_mode=mode))
            check(ref, got, t, mr.bits(t) > 8)


def test_round_to_multiple_options_errors():
    with pytest.raises(pa.ArrowInvalid, match="Integer value 1000 not in range: -128 to 127"):
        pc.round_to_multiple(pa.array([1], pa.int8()), multiple=1000)
    with pytest.raises(pa.ArrowInvalid, match="Rounding multiple must be positive"):
        pc.round_to_multiple(pa.array([1], pa.int8()), multiple=0)
    with pytest.raises(pa.ArrowInvalid, match="Rounding to -3 digits is out of range for type int8"):
        pc.round(pa.array([1], pa.int8()), -3)


# ---------------------------------------------------------------------------------------------------------------------
def kat_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", kat_cases(), ids=lambda c: c["id"])
def test_kat(case):
    t, fn, args = case["type"], case["function"], case.get("options", {})
    case = dict(case, x=[float(v) if isinstance(v, str) else v for v in case["x"]])
    if fn in mr.UNARY:
        ref = run_ref(lambda: mr.unary(fn, case["x"], t)[0])
    elif fn in mr.BINARY:
        ref = run_ref(lambda: mr.binary(fn, case["x"], case["y"], t))
    elif fn == "round":
        ref = run_ref(lambda: mr.round_(case["x"], t, args.get("ndigits", 0), args.get("round_mode", "half_to_even")))
    elif fn == "round_to_multiple":
        ref = run_ref(lambda: mr.round_to_multiple(case["x"], t, args["multiple"], args.get("round_mode", "half_to_even")))
    else:
        ref = run_ref(lambda: mr.round_binary(case["x"], t, case["y"], args.get("round_mode", "half_to_even")))
    if "error" in case:
        assert ref[0] == "Invalid" and case["error"] in ref[1]
    else:
        assert ref[0] == "ok", ref
        want = [None if v is None else (float(v) if isinstance(v, str) else v) for v in case["expected"]]
        same(to_py(ref[1], t), want, t)
