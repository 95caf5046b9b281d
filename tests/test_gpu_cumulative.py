"""The device's cumulative functions against tests/cumulative_ref.py: every function over the ten types with and without
a start, in both null modes; lengths around the 4096-row scan tile; bit offsets 1-63; chunked columns with empty chunks,
unaligned chunk edges and an early null; launches per call; both options forms of call_function; float min / max bit
for bit; float sums, products and means exactly on data whose partial results are representable and within the
sequential fold's error bound on random data; and a 1B-row column whose only overflow, or only null, is in its last
rows, so the look-back chain is deep."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import cumulative_ref as cr
from tests.test_cumulative_oracle import bits_equal

pytestmark = pytest.mark.gpu

TILE = 4096
LENGTHS = [0, 1, 63, TILE - 1, TILE, TILE + 1, 5 * TILE + 17]


def column(t: pa.DataType, n: int, seed: int, null_frac=0.1, offset=0, name="cumulative_sum") -> pa.Array:
    """n values of t sliced at `offset`, chosen so that every fold order gives the same bits: full-range integers for
    sums (wrapping is exact anyway), integers below 1000 and quarter-integers for means and float sums (partial sums
    stay exact), and +-1 with a few 2 / +-0.5 for float products (partial products are powers of two inside the
    exponent range)"""
    rng = np.random.default_rng(seed)
    m = n + offset
    dt = np.dtype(t.to_pandas_dtype())
    if dt.kind == "f" and "prod" in name:
        vals = rng.choice(np.array([1.0, -1.0, 2.0, 0.5, -0.5], dt), m, p=[0.49, 0.49, 0.01, 0.005, 0.005])
    elif dt.kind == "f" and name in ("cumulative_min", "cumulative_max"):
        vals = rng.choice(np.array([0.0, -0.0, 1.5, -1.5, np.inf, -np.inf, np.nan, 3.0], dt), m)
        vals = np.where(rng.random(m) < 0.5, vals, rng.integers(-1000, 1000, m).astype(dt))
    elif dt.kind == "f":
        vals = (rng.integers(-64, 64, m) / 4).astype(dt)
    elif name == "cumulative_mean":  # sums of these stay below 2^53, exact in double in any order
        vals = rng.integers(0 if dt.kind == "u" else -1000, 1000, m).astype(dt)
    elif "checked" in name and "sum" in name:  # full range would overflow at once: keep most columns valid
        vals = rng.integers(0 if dt.kind == "u" else -3, 4, m).astype(dt)
    elif "prod" in name:
        vals = rng.choice(np.array([1, 1, 1, 2, 3, 0] + ([255 if dt.kind == "u" else -1]), dt), m)
    else:
        info = np.iinfo(dt)
        vals = rng.integers(int(info.min), int(info.max), m, dtype=dt, endpoint=True)
    mask = rng.random(m) < null_frac if null_frac else None
    return pa.array(vals, t, mask=mask).slice(offset)


def expect(name, chunks, start=None, skip_nulls=False, ctx=None):
    """the device result over the pyarrow chunks equals the restatement bit for bit, or both raise overflow"""
    dev = [DeviceArray.from_arrow(c, ctx) for c in chunks]
    arg = dev[0] if len(dev) == 1 else dev
    try:
        want = cr.cumulative(name, chunks, start, skip_nulls)
    except cr.Overflow:
        with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
            getattr(bc, name)(arg, start=start, skip_nulls=skip_nulls)
        return None
    got = getattr(bc, name)(arg, start=start, skip_nulls=skip_nulls)
    assert got.null_count == want.null_count
    assert bits_equal(got.to_arrow(), want), (name, start, skip_nulls)
    return got


@pytest.mark.parametrize("t", cr.TYPES, ids=str)
@pytest.mark.parametrize("name", cr.FUNCTIONS)
def test_every_function_type_and_option(ctx, name, t):
    seed = zlib.crc32(f"{name}-{t}".encode())
    for i, n in enumerate(LENGTHS):
        for skip_nulls in (False, True):
            for start in (None, 3):
                for null_frac in (0.0, 0.001, 0.2):
                    expect(name, [column(t, n, seed + i, null_frac, name=name)], start, skip_nulls, ctx)


@pytest.mark.parametrize("name", cr.FUNCTIONS)
def test_bit_offsets(ctx, name):
    for t in (pa.int8(), pa.uint32(), pa.int64(), pa.float64()):
        for offset in range(1, 64):
            for skip_nulls in (False, True):
                expect(name, [column(t, 300 + offset, offset, 0.05, offset, name)], None, skip_nulls, ctx)


@pytest.mark.parametrize("name", cr.FUNCTIONS)
def test_chunks(ctx, name):
    for t in (pa.int16(), pa.int64(), pa.uint64(), pa.float32(), pa.float64()):
        sizes = [0, 100, 0, 4095, 1, 64, 8193, 0, 77, 3 * TILE + 5]
        seed = zlib.crc32(f"{name}-{t}-chunks".encode())
        base = column(t, sum(sizes) + 3, seed, 0.0, name=name)
        chunks, o = [], 3
        for s in sizes:
            chunks.append(base.slice(o, s))
            o += s
        for skip_nulls in (False, True):
            for start in (None, 2):
                expect(name, chunks, start, skip_nulls, ctx)
        # a null in an early chunk nulls every later row under skip_nulls=False
        with_null = [chunks[0], chunks[1], pa.array([None] + chunks[3].to_pylist()[1:], t)] + chunks[4:]
        got = expect(name, with_null, None, False, ctx)
        if got is not None:
            assert got.null_count == sum(sizes) - 100
        expect(name, with_null, None, True, ctx)
        # nullable chunks whose output starts inside a validity word
        nullable = [column(t, s, seed + k, 0.1, k % 7, name) for k, s in enumerate(sizes)]
        for skip_nulls in (False, True):
            expect(name, nullable, None, skip_nulls, ctx)


def test_mean_across_chunks(ctx):
    rng = np.random.default_rng(11)
    for t in (pa.int32(), pa.uint8(), pa.float32()):
        chunks = [pa.array(rng.integers(0, 100, s).astype(t.to_pandas_dtype()), t, mask=rng.random(s) < 0.1)
                  for s in (5, 0, 4097, 63, 20000)]
        for skip_nulls in (False, True):
            expect("cumulative_mean", chunks, None, skip_nulls, ctx)
        # start is cast (and so checked) but ignored
        expect("cumulative_mean", chunks, 50, True, ctx)


def test_float_min_max_bits(ctx):
    for t in (pa.float32(), pa.float64()):
        got = bc.cumulative_min(DeviceArray.from_arrow(pa.array([0.0, -0.0, 0.0], t), ctx)).to_arrow()
        assert np.signbit(np.asarray(got)).tolist() == [False, True, False]
        got = bc.cumulative_max(DeviceArray.from_arrow(pa.array([-0.0, 0.0, -0.0], t), ctx), start=-0.0).to_arrow()
        assert np.signbit(np.asarray(got)).tolist() == [True, False, True]
        smallest = np.finfo(t.to_pandas_dtype()).smallest_normal
        assert bc.cumulative_max(DeviceArray.from_arrow(pa.array([-5.0], t), ctx)).to_arrow().to_pylist() == [smallest]
        biggest = float(np.finfo(t.to_pandas_dtype()).max)
        assert bc.cumulative_min(DeviceArray.from_arrow(pa.array([float("inf")], t), ctx)).to_arrow().to_pylist() == [biggest]
        # NaN is ignored on either side; across a tile edge too
        vals = [float("nan")] * (TILE + 3) + [2.0, float("nan"), -0.0, 0.0]
        for name in ("cumulative_min", "cumulative_max"):
            for start in (None, float("nan")):
                expect(name, [pa.array(vals, t)], start, False, ctx)


def test_float_specials_exact(ctx):
    rng = np.random.default_rng(5)
    for t in (pa.float32(), pa.float64()):
        for name in ("cumulative_sum", "cumulative_prod", "cumulative_mean"):
            for _ in range(4):
                vals = rng.choice([1.0, -1.0, 2.0, 0.0, -0.0, float("inf"), float("-inf"), float("nan")], 9000,
                                  p=[0.3, 0.3, 0.2, 0.05, 0.05, 0.04, 0.04, 0.02])
                # every other scale factor is 0.5, so any run of rows multiplies to 2^-1, 2^0 or 2^1: no partial
                # product leaves the exponent range in any fold order
                scale = np.flatnonzero(vals == 2.0)
                vals[scale[1::2]] = 0.5
                expect(name, [pa.array(vals, t, mask=rng.random(9000) < 0.05)], None, True, ctx)


@pytest.mark.parametrize("t", [pa.float32(), pa.float64()], ids=str)
def test_float_sums_within_the_sequential_bound(ctx, t):
    """random data: |device - exact| <= n * eps * sum|x| at every row, the bound the sequential fold also has"""
    rng = np.random.default_rng(3)
    n = 200_000
    dt = np.dtype(t.to_pandas_dtype())
    vals = rng.standard_normal(n).astype(dt)
    eps = float(np.finfo(dt).eps)
    exact = np.cumsum(vals.astype(np.longdouble))
    bound = np.arange(1, n + 1) * eps * np.cumsum(np.abs(vals).astype(np.longdouble))
    got = np.asarray(bc.cumulative_sum(DeviceArray.from_arrow(pa.array(vals, t), ctx)).to_arrow()).astype(np.longdouble)
    assert (np.abs(got - exact) <= bound).all()
    mean = np.asarray(bc.cumulative_mean(DeviceArray.from_arrow(pa.array(vals, t), ctx)).to_arrow()).astype(np.longdouble)
    exact_mean = np.cumsum(vals.astype(np.longdouble)) / np.arange(1, n + 1)
    mbound = np.arange(1, n + 1) * 2.0 ** -52 * np.cumsum(np.abs(vals).astype(np.longdouble)) / np.arange(1, n + 1)
    assert (np.abs(mean - exact_mean) <= mbound + 1e-300).all()
    pvals = rng.uniform(0.999, 1.001, n).astype(dt)
    got = np.asarray(bc.cumulative_prod(DeviceArray.from_arrow(pa.array(pvals, t), ctx)).to_arrow()).astype(np.longdouble)
    exact = np.cumprod(pvals.astype(np.longdouble))
    assert (np.abs(got - exact) <= np.arange(1, n + 1) * eps * np.abs(exact) * 1.01).all()


def test_checked_overflow_deep_in_a_long_column(ctx):
    n = 3 * 10 ** 6
    for pos in (5, TILE - 1, TILE, 77 * TILE + 13, n - 1):
        vals = np.ones(n, np.int64)
        vals[pos] = np.iinfo(np.int64).max
        arr = pa.array(vals)
        with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
            bc.cumulative_sum_checked(DeviceArray.from_arrow(arr, ctx))
        # after a null under skip_nulls=False the row is not combined
        masked = pa.array(vals, mask=np.arange(n) == pos - 1 if pos else None)
        expect("cumulative_sum_checked", [masked], None, False, ctx)
        pvals = np.ones(n, np.int32)
        pvals[pos] = 1 << 20
        pvals[(pos + 9) % n] = 1 << 11
        expect("cumulative_prod_checked", [pa.array(pvals)], None, False, ctx)
    # [2^62, 4, 0] raises though the final product is 0
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.cumulative_prod_checked(DeviceArray.from_arrow(pa.array([2 ** 62, 4, 0]), ctx))
    # [1, null, 2^62, 2^62] does not: the overflow is after the first null
    got = bc.cumulative_sum_checked(DeviceArray.from_arrow(pa.array([1, None, 2 ** 62, 2 ** 62]), ctx))
    assert got.to_arrow().to_pylist() == [1, None, None, None]


def test_starts_and_types(ctx):
    x = DeviceArray.from_arrow(pa.array([1, 2], pa.int64()), ctx)
    with pytest.raises(pa.ArrowInvalid, match="Float value 1.500000 was truncated converting to int64"):
        bc.cumulative_sum(x, start=1.5)
    with pytest.raises(pa.ArrowInvalid, match="Integer value 1000 not in range: -128 to 127"):
        bc.cumulative_sum(DeviceArray.from_arrow(pa.array([1], pa.int8()), ctx), start=1000)
    assert bc.cumulative_sum(x, start=pa.scalar(None, pa.int64())).to_arrow().to_pylist() == [1, 3]
    assert bc.cumulative_mean(x, start=100).to_arrow().to_pylist() == [1.0, 1.5]
    with pytest.raises(pa.ArrowInvalid, match="Float value 1.500000 was truncated converting to int64"):
        bc.cumulative_mean(x, start=1.5)
    with pytest.raises(pa.ArrowNotImplementedError, match="Function 'cumulative_sum' has no kernel matching input types"):
        bc.cumulative_sum(DeviceArray.from_arrow(pa.array([True]), ctx))


def test_launches_per_call(ctx):
    chunks = [DeviceArray.from_arrow(pa.array(np.arange(s, dtype=np.int64)), ctx) for s in (5, 0, 10000, 3)]
    for arg, want in ((chunks[0], 1), (chunks, 3), (chunks[1], 0)):
        before = _cabi.lib().b2_launch_count()
        bc.cumulative_sum(arg)
        assert _cabi.lib().b2_launch_count() - before == want


def test_call_function_options(ctx):
    import pyarrow.compute as pc
    x = DeviceArray.from_arrow(pa.array([3, None, 1, 2], pa.int64()), ctx)
    for name in cr.FUNCTIONS:
        want = getattr(bc, name)(x, skip_nulls=True).to_arrow()
        assert bc.call_function(name, [x], pc.CumulativeOptions(skip_nulls=True)).to_arrow().equals(want)
        assert bc.call_function(name, [x], {"skip_nulls": True}).to_arrow().equals(want)
        want = getattr(bc, name)(x, start=5).to_arrow()
        assert bc.call_function(name, [x], {"start": 5}).to_arrow().equals(want)
        with pytest.raises(pa.ArrowNotImplementedError, match="as a dict"):
            bc.call_function(name, [x], pc.CumulativeOptions(start=5))
    assert set(cr.FUNCTIONS) <= set(bc.list_functions())


N_BIG = 1_000_000_000


def test_one_billion_rows(ctx):
    """one overflow, or one null, in the last rows of 1B: every tile's state travels the whole look-back chain"""
    import torch
    from tests.test_gpu_fullsize import as_tensor
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()
    if torch.cuda.mem_get_info()[0] < 20 * N_BIG:
        pytest.skip("needs ~20 GB of free device memory")

    def equals_arange(out, rows):
        """out[:rows] == 1, 2, ..., rows, compared in slices so that no second 8 GB tensor is made"""
        got = as_tensor(torch, out, torch.int64)
        step = 1 << 27
        return all(torch.equal(got[lo:min(lo + step, rows)], torch.arange(lo + 1, min(lo + step, rows) + 1,
                                                                             dtype=torch.int64, device="cuda"))
                   for lo in range(0, rows, step))
    vals = torch.ones(N_BIG, dtype=torch.int64, device="cuda")
    x = DeviceArray.from_pointers(ctx, pa.int64(), N_BIG, vals.data_ptr())
    torch.cuda.synchronize()
    out = bc.cumulative_sum_checked(x)
    ctx.sync()
    assert out.null_count == 0 and equals_arange(out, N_BIG)
    del out
    vals[N_BIG - 2] = 2 ** 63 - N_BIG + 1  # the prefix reaches INT64_MAX there, and overflows on the last row
    torch.cuda.synchronize()
    with pytest.raises(pa.ArrowInvalid, match="^overflow$"):
        bc.cumulative_sum_checked(x)
    vals[N_BIG - 2] = 1
    # the only null, three rows from the end
    bits = torch.full(((N_BIG + 7) // 8 + 64,), 0xFF, dtype=torch.uint8, device="cuda")
    bits[(N_BIG - 3) // 8] &= ~(1 << ((N_BIG - 3) % 8)) & 0xFF
    xn = DeviceArray.from_pointers(ctx, pa.int64(), N_BIG, vals.data_ptr(), validity_ptr=bits.data_ptr(), null_count=1)
    torch.cuda.synchronize()
    out = bc.cumulative_sum(xn)
    ctx.sync()
    assert out.null_count == 3
    assert equals_arange(out, N_BIG - 3)
    del out
    out = bc.cumulative_max(xn, skip_nulls=True)
    ctx.sync()
    assert out.null_count == 1
