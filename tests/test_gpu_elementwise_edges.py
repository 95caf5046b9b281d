"""Cast, arithmetic, comparison, if_else and the fused take + cast + arithmetic at the edges where kernels go wrong, against
the EXACT references of tests/elementwise_ref.py (pinned to the reference binary by test_elementwise_edges_oracle.py):
full-range integers and their boundaries, NaN of several payloads, +-0, +-inf, subnormals, the largest finite values and the
float32 rounding edges (ties, the overflow threshold, results that underflow).  Results compare with exact_ref.assert_same
(bit-exact on valid slots, any NaN equal to any NaN), selections (if_else) bit for bit; errors by type and text.

The special rows sit both in the vectorised main loop and in the scalar tail of the streaming kernels (elementwise.cuh:
lengths of k * (32 * V * kUnroll) +- 1, and offsets that make the 16-byte loads impossible), and one 1-byte case runs past
map_grid's CTA cap so the grid-stride loop takes a second turn."""
import itertools
import math
import os
import re

import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import elementwise_ref as ew
from tests import exact_ref as er
from tests.elementwise_ref import edges
from tests.test_elementwise_edges_oracle import bits_equal, outcome, same_outcome, same_result
from tests.util import SEED

pytestmark = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_b200", "csrc")


def _constant(text, name):
    return int(re.search(rf"constexpr int {name} = (\d+);", text).group(1))


def kernel_constants():
    """kUnroll, kWarpsPerBlock and map_grid's CTA cap, read from the kernel sources"""
    with open(os.path.join(CSRC, "common.cuh")) as f:
        common = f.read()
    with open(os.path.join(CSRC, "elementwise.cuh")) as f:
        ew_src = f.read()
    block, sms = _constant(common, "kBlock"), _constant(common, "kSMs")
    cap = re.search(r"return grid_for\(n, kTile, kSMs \* (\d+) \* (\d+)\);", ew_src)
    return _constant(ew_src, "kUnroll"), block // 32, sms * int(cap.group(1)) * int(cap.group(2))


UNROLL, WARPS, CTA_CAP = kernel_constants()


def warp_tile(t: pa.DataType) -> int:
    """elements one warp covers per step of map2_kernel / compare_kernel: 32 lanes x V = 16 / width x kUnroll"""
    return 32 * (16 // (t.bit_width // 8)) * UNROLL


def dev(x, ctx):
    return DeviceArray.from_arrow(x, ctx) if isinstance(x, pa.Array) else x


def random_values(t: pa.DataType, n: int, rng) -> list:
    """full range: uniform integers, or floats with uniformly random bit patterns (every exponent, NaNs rarely)"""
    if pa.types.is_integer(t):
        lo, hi = ew.int_range(t)
        return [int(v) for v in rng.integers(lo, hi, n, dtype=ew.np_dtype(t), endpoint=True)]
    u = np.uint32 if t == pa.float32() else np.uint64
    return rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(ew.np_dtype(t)).astype(np.float64).tolist()


def special_pairs(tl, tr, n, rng, offset=0):
    """two arrays of n rows (sliced at `offset`) whose first and last rows hold every pair of edge values, the rest full
    range; about one row in ten is null on each side"""
    rows = list(itertools.product(edges(tl), edges(tr)))
    m = n + offset
    assert m >= 2 * len(rows)
    left, right = random_values(tl, m, rng), random_values(tr, m, rng)
    for k, (a, b) in enumerate(rows):
        left[offset + k], right[offset + k] = a, b
        left[m - len(rows) + k], right[m - len(rows) + k] = a, b
    lv, rv = rng.random(m) > 0.1, rng.random(m) > 0.1
    return ew.to_array(left, tl, lv).slice(offset), ew.to_array(right, tr, rv).slice(offset)


def length_for(t, pairs, plus: bool):
    tile = warp_tile(t)
    k = (2 * pairs + tile - 1) // tile + 1
    return k * tile + (1 if plus else -1)


def with_nulls(arr: pa.Array, extra: np.ndarray) -> pa.Array:
    """arr with the rows of `extra` null as well (the values under them unchanged)"""
    valid = er.valid_mask(arr) & ~extra
    return pa.Array.from_buffers(arr.type, len(arr), [pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()),
                                                      pa.py_buffer(er.raw(arr).tobytes())], null_count=int((~valid).sum()))


def failing_rows(op, left, right) -> np.ndarray:
    """the valid rows on which a checked op (or an integer division) fails"""
    n = len(left) if isinstance(left, pa.Array) else len(right)
    t = ew.common_numeric([left.type, right.type]) if left.type != right.type else left.type
    (a, va), (b, vb) = ew.promote(left, t, n), ew.promote(right, t, n)
    fn = ew.int_op if pa.types.is_integer(t) else ew.float_op
    return np.array([ok and fn(op, x, y, t)[1] is not None for x, y, ok in zip(a, b, va & vb)], bool)


def check_arith(ctx, op, left, right, msg):
    want = outcome(lambda: ew.arithmetic(op, left, right))
    got = outcome(lambda: getattr(bc, op)(dev(left, ctx), dev(right, ctx)).to_arrow())
    same_outcome(got, want, msg)
    if want[0] != "ok":
        # the same rows with the failing ones null: no error, and the values of the rest
        bad = failing_rows(op, left, right)
        assert bad.any(), msg
        if isinstance(left, pa.Array):
            left = with_nulls(left, bad)
        else:
            right = with_nulls(right, bad)
        want = outcome(lambda: ew.arithmetic(op, left, right))
        assert want[0] == "ok", msg
        same_outcome(outcome(lambda: getattr(bc, op)(dev(left, ctx), dev(right, ctx)).to_arrow()), want, msg + " (failing rows null)")


def scalar_choices(t):
    v = edges(t)
    if pa.types.is_integer(t):
        picks = [v[0], -1 if -1 in v else 0, v[-1]]
    else:
        picks = [math.nan, -0.0, math.inf, v[-3]]
    return [ew.to_array([x], t)[0] for x in picks]


# ---------------------------------------------------------------------------------------------------------------------
# arithmetic
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ew.NUMERIC, ids=str)
@pytest.mark.parametrize("op", ew.ARITH_OPS)
def test_arithmetic_edges(ctx, t, op):
    rng = np.random.default_rng(SEED + ew.NUMERIC.index(t) * 16 + ew.ARITH_OPS.index(op))
    pairs = len(edges(t)) ** 2
    for offset, plus in ((0, True), (1, False)):        # vectorised loop + scalar tail; then no 16-byte access at all
        n = length_for(t, pairs, plus)
        a, b = special_pairs(t, t, n, rng, offset)
        check_arith(ctx, op, a, b, f"{op} {t} array/array n={n} offset={offset}")
    n = length_for(t, len(edges(t)), True)
    tiled = ew.to_array((edges(t) * (n // len(edges(t)) + 1))[:n], t, rng.random(n) > 0.1).slice(3)
    for s in scalar_choices(t):
        check_arith(ctx, op, tiled, s, f"{op} {t} array/scalar {s}")
        check_arith(ctx, op, s, tiled, f"{op} {t} scalar/array {s}")
    null = pa.scalar(None, t)
    for left, right in ((a, null), (null, a)):
        got = getattr(bc, op)(dev(left, ctx), dev(right, ctx)).to_arrow()
        assert got.type == t and len(got) == len(a) and got.null_count == len(a)


@pytest.mark.parametrize("t", [pa.int8(), pa.int32(), pa.int64(), pa.uint64()], ids=str)
def test_checked_error_kind_is_the_last_offending_row(ctx, t):
    """divide_checked fails with "overflow" (INT_MIN / -1) or "divide by zero"; with both kinds in different CTAs the message is
    that of the last failing row, as in the reference"""
    lo, _ = ew.int_range(t)
    tile = warp_tile(t) * WARPS                            # rows per CTA
    n = 5 * tile + 7
    a = np.full(n, 9, ew.np_dtype(t))
    b = np.full(n, 2, ew.np_dtype(t))
    early, late = 3, 4 * tile + 5
    signed = pa.types.is_signed_integer(t)
    for first, second in (("overflow", "divide by zero"), ("divide by zero", "overflow")):
        if not signed and "overflow" in (first, second):
            continue
        x, y = a.copy(), b.copy()
        for row, kind in ((early, first), (late, second)):
            if kind == "overflow":
                x[row], y[row] = lo, -1
            else:
                y[row] = 0
        left, right = pa.array(x, t), pa.array(y, t)
        with pytest.raises(pa.ArrowInvalid, match=f"^{second}$"):
            ew.arithmetic("divide_checked", left, right)
        with pytest.raises(pa.ArrowInvalid, match=f"^{second}$"):
            bc.divide_checked(dev(left, ctx), dev(right, ctx))
        # the late row under a null: the early one speaks
        with pytest.raises(pa.ArrowInvalid, match=f"^{first}$"):
            bc.divide_checked(dev(left, ctx), dev(pa.array(y, t, mask=np.arange(n) == late), ctx))
    if not signed:
        y = b.copy()
        y[early] = y[late] = 0
        with pytest.raises(pa.ArrowInvalid, match="^divide by zero$"):
            bc.divide_checked(dev(pa.array(a, t), ctx), dev(pa.array(y, t), ctx))


def test_grid_stride_second_turn(ctx):
    """int8 past map_grid's CTA cap: the CTAs loop, and an error placed in the second turn is found"""
    tile = warp_tile(pa.int8()) * WARPS
    first_turn = CTA_CAP * tile
    n = first_turn + 3 * warp_tile(pa.int8()) + 5
    rng = np.random.default_rng(SEED)
    a = rng.integers(-60, 60, n, dtype=np.int8)
    b = rng.integers(-60, 60, n, dtype=np.int8)
    bad = first_turn + 1000 + int(rng.integers(0, 2 * warp_tile(pa.int8())))
    a[bad], b[bad] = 100, 100
    da, db = dev(pa.array(a), ctx), dev(pa.array(b), ctx)
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.add_checked(da, db)
    mask = np.zeros(n, bool)
    mask[bad] = True
    got = bc.add_checked(da, dev(pa.array(b, mask=mask), ctx)).to_arrow()
    want = (a.astype(np.int16) + b.astype(np.int16)).astype(np.int8)   # exact: no valid row overflows
    assert got.null_count == 1 and not got[bad].is_valid
    gv = er.raw(got)
    assert np.array_equal(np.delete(gv, bad), np.delete(want, bad))
    # divide_checked: overflow early in the first turn, a zero divisor in the second: the last one is reported
    b2 = np.where(b == 0, 1, b).astype(np.int8)
    a2 = a.copy()
    a2[bad] = 100
    a2[5], b2[5] = -128, -1
    b2[bad] = 0
    with pytest.raises(pa.ArrowInvalid, match="^divide by zero$"):
        bc.divide_checked(dev(pa.array(a2), ctx), dev(pa.array(b2), ctx))
    got = bc.divide(dev(pa.array(a2), ctx), dev(pa.array(b2, mask=mask), ctx)).to_arrow()
    a16, b16 = a2.astype(np.int16), np.where(b2 == 0, 1, b2).astype(np.int16)
    q = np.abs(a16) // np.abs(b16) * np.sign(a16) * np.sign(b16)       # truncated toward zero, exact in int16
    q[5] = 0                                                            # INT_MIN / -1
    assert np.array_equal(np.delete(er.raw(got), bad), np.delete(q.astype(np.int8), bad))


# ---------------------------------------------------------------------------------------------------------------------
# cast
# ---------------------------------------------------------------------------------------------------------------------
def cast_inputs(src, rng, offset):
    vals = edges(src)
    if src in (pa.int64(), pa.uint64()):
        vals = vals + [2 ** 60 + 2 ** 36 + 1, 2 ** 53 + 1, 2 ** 24 + 1, 2 ** 63 + 2 ** 39 + 1, 2 ** 64 - 2 ** 39]
        if src == pa.int64():
            vals = [v for v in vals if v < 2 ** 63] + [-(2 ** 60 + 2 ** 36 + 1), -(2 ** 53) - 1]
        else:
            vals = [v for v in vals if v >= 0]
    if src in (pa.int32(), pa.uint32()):
        vals = vals + [2 ** 24 + 1, 2 ** 24 + 3, 2 ** 31 - 1 if src == pa.int32() else 2 ** 32 - 1]
    if pa.types.is_floating(src):
        extra = [1.5, -2.5, 127.9, -128.9, 255.5, 1e10, -1e10, 2.0 ** 31, -(2.0 ** 31) - 1, 2.0 ** 32, 2.0 ** 63, -(2.0 ** 63),
                 2.0 ** 64, 5e9, -0.5, 65535.0, 65536.0]
        if src == pa.float64():
            extra += [1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, float(np.finfo(np.float32).max) + 2.0 ** 103,
                      float(np.finfo(np.float32).max) + 2.0 ** 103 - 2.0 ** 76, 2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -150,
                      2.0 ** -140, 1e-300, 2.0 ** 63 - 1024]
        vals = vals + [v if src == pa.float64() else float(np.float32(v)) for v in extra]
    n = length_for(src, len(vals), offset == 0)
    body = (vals * 2 + random_values(src, n + offset, rng))[:n + offset]
    body[n + offset - len(vals):] = vals                                # the tail too
    return ew.to_array(body, src, rng.random(n + offset) > 0.1).slice(offset)


@pytest.mark.parametrize("src", ew.NUMERIC, ids=str)
def test_cast_edges(ctx, src):
    rng = np.random.default_rng(SEED + 100 + ew.NUMERIC.index(src))
    for offset in (0, 1):
        x = cast_inputs(src, rng, offset)
        dx = dev(x, ctx)
        for dst in ew.NUMERIC:
            if dst == src:
                continue
            for safe in (True, False):
                msg = f"cast {src} -> {dst} safe={safe} offset={offset}"
                want = outcome(lambda: ew.cast(x, dst, safe))
                same_outcome(outcome(lambda: bc.cast(dx, dst, safe=safe).to_arrow()), want, msg)
                if want[0] != "ok":
                    bad = np.array([ok and ew.cast_value(v, src, dst, True)[1] is not None
                                    for v, ok in zip(ew.pylist(x), er.valid_mask(x))])
                    y = with_nulls(x, bad)
                    same_outcome(outcome(lambda: bc.cast(dev(y, ctx), dst, safe=True).to_arrow()),
                                 outcome(lambda: ew.cast(y, dst, True)), msg + " (failing rows null)")


# ---------------------------------------------------------------------------------------------------------------------
# compare
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", ew.NUMERIC, ids=str)
def test_compare_edges(ctx, t):
    rng = np.random.default_rng(SEED + 200 + ew.NUMERIC.index(t))
    pairs = len(edges(t)) ** 2
    cases = []
    for offset, plus in ((0, True), (3, False)):
        n = length_for(t, pairs, plus)
        cases.append(special_pairs(t, t, n, rng, offset))
    a37, b37 = special_pairs(t, t, 2 * pairs + 37, rng, 5)     # ends mid-word of the packed output
    cases.append((a37, b37))
    for left, right in cases:
        for s in scalar_choices(t) + [pa.scalar(None, t)]:
            for l, r in ((left, right), (left, s), (s, right)):
                for op in ew.COMPARE_OPS:
                    got = getattr(bc, op)(dev(l, ctx), dev(r, ctx)).to_arrow()
                    same_result(got, ew.compare(op, l, r), f"{op} {t} {l.type} {r.type} len={len(left)}")


MIXED = [
    # (left type, right type, left values, right values): the implicit safe cast to the common type must raise
    (pa.int64(), pa.uint64(), [1, -1, 0], [2 ** 63, 1, 2]),
    (pa.int64(), pa.uint64(), [1, -1, 0], [2 ** 64 - 1, 0, 2]),
    (pa.int64(), pa.float64(), [2 ** 53 + 1, 0, 1], [0.0, math.nan, -0.0]),
    (pa.int64(), pa.float64(), [-(2 ** 53) - 1, 0, 1], [1.0, 2.0, 3.0]),
    (pa.int32(), pa.float32(), [2 ** 24 + 1, 0, 1], [1.0, 2.0, 3.0]),
    (pa.uint32(), pa.float32(), [2 ** 25, 0, 1], [1.0, 2.0, 3.0]),
    # and where it succeeds
    (pa.int64(), pa.uint64(), [-1, 2 ** 63 - 1, 0], [2 ** 63 - 1, 5, 0]),
    (pa.int64(), pa.float64(), [2 ** 53, -(2 ** 53), 3], [math.nan, -0.0, 3.0]),
    (pa.int8(), pa.uint64(), [-128, 127, 0], [0, 127, 2 ** 63 - 1]),
]


@pytest.mark.parametrize("case", range(len(MIXED)))
def test_compare_and_arith_mixed_types(ctx, case):
    tl, tr, vl, vr = MIXED[case]
    reps = 200
    left = ew.to_array(vl * reps, tl)
    right = ew.to_array(vr * reps, tr)
    for l, r in ((left, right), (right, left), (left, right[len(vr) - 1]), (right[0], left), (left[0], right)):
        for op in ("less", "equal", "greater_equal"):
            same_outcome(outcome(lambda: getattr(bc, op)(dev(l, ctx), dev(r, ctx)).to_arrow()),
                         outcome(lambda: ew.compare(op, l, r)), f"{op} {l.type} {r.type}")
        for op in ("add", "subtract_checked"):
            same_outcome(outcome(lambda: getattr(bc, op)(dev(l, ctx), dev(r, ctx)).to_arrow()),
                         outcome(lambda: ew.arithmetic(op, l, r)), f"{op} {l.type} {r.type}")
        c = pa.array(np.arange(len(left)) % 2 == 0)
        same_outcome(outcome(lambda: bc.if_else(dev(c, ctx), dev(l, ctx), dev(r, ctx)).to_arrow()),
                     outcome(lambda: ew.if_else(c, l, r)), f"if_else {l.type} {r.type}")


# ---------------------------------------------------------------------------------------------------------------------
# if_else
# ---------------------------------------------------------------------------------------------------------------------
IF_ELSE_PAIRS = [(t, t) for t in ew.NUMERIC] + [
    (pa.int8(), pa.uint8()), (pa.int32(), pa.uint32()), (pa.uint16(), pa.float32()), (pa.int32(), pa.float64()),
    (pa.float32(), pa.float64()), (pa.int64(), pa.uint8()), (pa.uint32(), pa.int64())]


@pytest.mark.parametrize("tl,tr", IF_ELSE_PAIRS, ids=lambda t: str(t))
def test_if_else_edges(ctx, tl, tr):
    rng = np.random.default_rng(SEED + 300)
    if tl != tr:   # values every promotion admits
        def ok(v, t):
            return math.isnan(v) or not math.isinf(v) and abs(v) <= 2 ** 24 if isinstance(v, float) else \
                ew.cast_value(v, t, ew.common_numeric([tl, tr]), True)[1] is None
        vl, vr = [v for v in edges(tl) if ok(v, tl)], [v for v in edges(tr) if ok(v, tr)]
        rows = list(itertools.product(vl, vr))
        n = len(rows) * 3 + 1
        left = ew.to_array([r[0] for r in rows] * 3 + [vl[0]], tl, rng.random(n) > 0.1)
        right = ew.to_array([r[1] for r in rows] * 3 + [vr[0]], tr, rng.random(n) > 0.1)
    else:
        left, right = special_pairs(tl, tr, length_for(tl, len(edges(tl)) ** 2, True), rng, 0)
        n = len(left)
    cond = pa.array(rng.random(n + 3) < 0.5, mask=rng.random(n + 3) < 0.1).slice(3)
    scal_l = [ew.to_array([v], tl)[0] for v in (edges(tl)[:2] if tl != tr else [edges(tl)[3], edges(tl)[-1]])] + [pa.scalar(None, tl)]
    scal_r = [ew.to_array([v], tr)[0] for v in edges(tr)[2:4]] + [pa.scalar(None, tr)]
    shapes = [(left, right)] + [(left, s) for s in scal_r] + [(s, right) for s in scal_l]
    for c in (cond, pa.scalar(True), pa.scalar(False), pa.scalar(None, pa.bool_())):
        for l, r in shapes:
            msg = f"if_else {l.type} {r.type} cond={c.type if isinstance(c, pa.Array) else c}"
            want = ew.if_else(c, l, r)
            got = bc.if_else(dev(c, ctx), dev(l, ctx), dev(r, ctx)).to_arrow()
            (bits_equal if tl == tr else er.assert_same)(got, want, msg)


# ---------------------------------------------------------------------------------------------------------------------
# fused take + cast + add / subtract / multiply
# ---------------------------------------------------------------------------------------------------------------------
F32_MAX = float(np.finfo(np.float32).max)


def fused_values(vt):
    """the values a take + cast must convert exactly"""
    if vt == pa.float64():
        return ([float(v) for v in er.special_values(np.float64)] +
                [1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, -(1 + 2.0 ** -24), F32_MAX + 2.0 ** 103, F32_MAX + 2.0 ** 103 - 2.0 ** 76,
                 -(F32_MAX + 2.0 ** 103), 2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -150, 2.0 ** -140, 1e-300, 1.7976931348623157e308,
                 2.0 ** 24 + 1, 0.1, 1.0, -1.0])
    if vt == pa.float32():
        return [float(v) for v in er.special_values(np.float32)] + [F32_MAX, -F32_MAX, 1.0, float(np.float32(0.1))]
    lo, hi = ew.int_range(vt)
    v = [lo, hi, lo + 1, hi - 1, 0, -1, 1, 2 ** 24 + 1, 2 ** 24 + 3, -(2 ** 24) - 1, 2 ** 31 - 1]
    if vt == pa.int64():
        v += [2 ** 60 + 2 ** 36 + 1, -(2 ** 60 + 2 ** 36 + 1), 2 ** 53 + 1, 2 ** 62 + 2 ** 38, 2 ** 63 - 2 ** 39]
    return [x for x in v if lo <= x <= hi]


def fused_others(to):
    big = F32_MAX if to == pa.float32() else 1.7976931348623157e308
    return [0.0, -0.0, math.inf, -math.inf, math.nan, 1.0, -1.0, big, 2.0 ** -149]


@pytest.mark.parametrize("vt", [pa.float64(), pa.float32(), pa.int64(), pa.int32()], ids=str)
@pytest.mark.parametrize("to", [pa.float32(), pa.float64()], ids=str)
def test_fused_take_cast_arith_edges(ctx, monkeypatch, vt, to):
    rng = np.random.default_rng(SEED + 400)
    specials = fused_values(vt)
    others = fused_others(to)
    n_v = len(specials) + 3000
    vals = specials + random_values(vt, n_v - len(specials), rng)
    vvalid = rng.random(n_v) > 0.05
    vvalid[:len(specials)] = True
    values = ew.to_array(vals, vt, vvalid)
    rows = list(itertools.product(range(len(specials)), others))        # every special value against every special `other`
    tile = 32 * 2 * UNROLL                                              # 8-byte indices: V = 2
    n = ((2 * len(rows)) // tile + 2) * tile + 1
    idx = rng.integers(0, n_v, n).tolist()
    oth = [ew.f64_to_f32(v) if to == pa.float32() else v for v in random_values(pa.float64(), n, rng)]
    for k, (j, o) in enumerate(rows):
        idx[k], oth[k] = j, o
        idx[n - len(rows) + k], oth[n - len(rows) + k] = j, o
    ivalid, ovalid = rng.random(n) > 0.05, rng.random(n) > 0.05
    for it in (pa.int64(), pa.uint32()):
        indices = pa.array(np.array(idx, ew.np_dtype(it)), it, mask=~ivalid)
        other = ew.to_array(oth, to, ovalid)
        dv, di, do = dev(values, ctx), dev(indices, ctx), dev(other, ctx)
        for op in ("add", "subtract", "multiply"):
            want = ew.take_cast_arith(values, indices, to, op, other)
            for partition in ("0", "1"):
                monkeypatch.setenv("B2_TAKE_PARTITION", partition)
                if partition == "1":
                    monkeypatch.setenv("B2_TAKE_PART_BAND_KB", "1")
                else:
                    monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
                got = bc.take_cast_arith(dv, di, to, op, do).to_arrow()
                er.assert_same(got, want, msg=f"{vt} -> {to} {op} idx {it} partition={partition}")
                assert got.null_count == want.null_count
        # a scalar `other`: NaN, -0.0 and inf
        for s in (math.nan, -0.0, -math.inf):
            sc = ew.to_array([s], to)[0]
            want = ew.take_cast_arith(values, indices, to, "add", sc)
            for partition in ("0", "1"):
                monkeypatch.setenv("B2_TAKE_PARTITION", partition)
                monkeypatch.setenv("B2_TAKE_PART_BAND_KB", "1")
                er.assert_same(bc.take_cast_arith(dv, di, to, "add", sc).to_arrow(), want, msg=f"scalar {s} partition={partition}")


def test_fused_signed_zero_and_infinity_sums(ctx, monkeypatch):
    """-0 + -0 = -0, +0 + -0 = +0, inf + -inf = NaN, and -0 * +x = -0 through both paths"""
    values = pa.array([-0.0, 0.0, math.inf, -math.inf, 1.0])
    indices = pa.array([0, 1, 2, 3, 0, 4, 1], pa.int64())
    other = pa.array([-0.0, -0.0, -math.inf, math.inf, 0.0, -0.0, 5.0], pa.float32())
    want_add = [-0.0, 0.0, math.nan, math.nan, 0.0, 1.0, 5.0]
    want_mul = [0.0, -0.0, -math.inf, -math.inf, -0.0, -0.0, 0.0]
    for partition in ("0", "1"):
        monkeypatch.setenv("B2_TAKE_PARTITION", partition)
        monkeypatch.setenv("B2_TAKE_PART_BAND_KB", "1")
        for op, w in (("add", want_add), ("multiply", want_mul)):
            got = bc.take_cast_arith(dev(values, ctx), dev(indices, ctx), pa.float32(), op, dev(other, ctx)).to_arrow()
            er.assert_same(got, pa.array(w, pa.float32()), msg=f"{op} partition={partition}")
            er.assert_same(got, ew.take_cast_arith(values, indices, pa.float32(), op, other), msg=f"{op} exact_ref")
