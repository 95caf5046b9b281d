"""hash_variance / hash_stddev / hash_skew / hash_kurtosis and the ungrouped variance / stddev / skew / kurtosis on the
device: the exact path bit for bit against Fractions, the two-pass path within a bound computed from the data, special
floats and null rules against pyarrow, and run-to-run reproducibility of the ungrouped result."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import exact_ref as er
from tests import moments_ref as mr
from tests.test_gpu_aggregate_edges import REGIMES
from tests.util import SEED

pytestmark = pytest.mark.gpu
NARROW = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32()]
SAMPLE = 1500  # groups checked exactly per run in the large regimes


def dev(a, ctx):
    return DeviceArray.from_arrow(a, ctx)


def run(ctx, fn, vals, ids, groups, merged=False, **opts):
    """one aggregator over all rows, or (merged) two partial states -- the second with its ids reversed -- merged back"""
    agg = bc.HashAggregator(fn, vals.type, ctx=ctx, **opts)
    agg.resize(groups)
    if not merged:
        agg.consume(dev(vals, ctx), dev(pa.array(ids, pa.uint32()), ctx))
        return agg.finalize().to_arrow()
    h = len(ids) // 2
    agg.consume(dev(vals.slice(0, h), ctx), dev(pa.array(ids[:h], pa.uint32()), ctx))
    other = bc.HashAggregator(fn, vals.type, ctx=ctx, **opts)
    other.resize(groups)
    other.consume(dev(vals.slice(h), ctx), dev(pa.array((groups - 1 - ids[h:]).astype(np.uint32)), ctx))
    agg.merge(other, dev(pa.array(np.arange(groups - 1, -1, -1, dtype=np.uint32)), ctx))
    return agg.finalize().to_arrow()


def full_range(t, n, rng, nulls=0.05):
    info = np.iinfo(t.to_pandas_dtype())
    v = rng.integers(int(info.min), int(info.max), n, dtype=np.int64, endpoint=True)
    # the extremes themselves, in every group
    v[: n // 50] = int(info.min)
    v[n // 50: n // 25] = int(info.max)
    rng.shuffle(v)
    return pa.array(v.astype(t.to_pandas_dtype()), t, mask=rng.random(n) < nulls)


def exact_groups(vals: pa.Array, ids, groups, check):
    """per checked group: (count, saw_null, S1, S2) as Python ints"""
    ok = np.asarray(vals.is_valid().to_numpy(zero_copy_only=False), bool)
    x = np.asarray(vals.to_numpy(zero_copy_only=False)).astype(np.int64)
    x = np.where(ok, x, 0)
    order = np.argsort(ids, kind="stable")
    starts = np.searchsorted(ids[order], np.arange(groups + 1))
    out = {}
    for g in check:
        rows = order[starts[g]:starts[g + 1]]
        xs = [int(v) for v in x[rows][ok[rows]]]
        out[g] = (len(xs), not ok[rows].all(), sum(xs), sum(v * v for v in xs))
    return out


def expect_exact(fn, stats, ddof, skip_nulls, min_count):
    n, saw, s1, s2 = stats
    if mr.is_null(fn, n, saw, ddof, skip_nulls, min_count):
        return None
    v = float(mr.Fraction(n * s2 - s1 * s1, n * (n - ddof)))
    return math.sqrt(v) if fn == "stddev" else v


OPTION_GRID = [(0, True, 0), (1, True, 5), (2, False, 0), (1, False, 1)]


@pytest.mark.parametrize("regime", ["private", "atomic", "banded", "merge"])
@pytest.mark.parametrize("t", NARROW, ids=str)
def test_exact_path_bit_for_bit(ctx, t, regime):
    groups, n = REGIMES["atomic" if regime == "merge" else regime]
    rng = np.random.default_rng(SEED + groups + NARROW.index(t))
    ids = rng.integers(0, groups, n).astype(np.uint32)
    ids[:10] = 0  # a group that surely has rows
    vals = full_range(t, n, rng)
    check = range(groups) if groups <= SAMPLE else rng.choice(groups, SAMPLE, replace=False)
    stats = exact_groups(vals, ids, groups, check)
    for fn in ("variance", "stddev"):
        for ddof, skip_nulls, min_count in OPTION_GRID:
            got = run(ctx, "hash_" + fn, vals, ids, groups, merged=regime == "merge", ddof=ddof, skip_nulls=skip_nulls,
                      min_count=min_count)
            assert got.type == pa.float64()
            for g in check:
                want = expect_exact(fn, stats[g], ddof, skip_nulls, min_count)
                assert got[int(g)].as_py() == want, (fn, t, regime, ddof, skip_nulls, min_count, int(g))


@pytest.mark.parametrize("t", NARROW, ids=str)
def test_exact_path_ungrouped(ctx, t):
    rng = np.random.default_rng(SEED + 3)
    chunks = [full_range(t, n, rng) for n in (1 << 18, 1000, 0, 77)]
    n, saw, s1, s2 = 0, False, 0, 0
    for c in chunks:
        st = exact_groups(c, np.zeros(len(c), np.uint32), 1, [0])[0]
        n, saw, s1, s2 = n + st[0], saw or st[1], s1 + st[2], s2 + st[3]
    dchunks = [dev(c, ctx) for c in chunks]
    for fn in ("variance", "stddev"):
        for ddof, skip_nulls, min_count in OPTION_GRID:
            want = expect_exact(fn, (n, saw, s1, s2), ddof, skip_nulls, min_count)
            got = getattr(bc, fn)(dchunks, ddof=ddof, skip_nulls=skip_nulls, min_count=min_count)
            assert got.type == pa.float64() and got.as_py() == want, (fn, t, ddof, skip_nulls, min_count)
            one = getattr(bc, fn)(dev(pa.concat_arrays(chunks), ctx), ddof=ddof, skip_nulls=skip_nulls, min_count=min_count)
            assert one.as_py() == want


def test_exact_path_carries_past_64_bits(ctx):
    """17 consumes of 2^28 int32 rows near +-2^31 in three groups (about 1.5e9 rows per group), merged with a second
    state: Sx^2 passes 2^64 many times over, the 128-bit limbs carry, the result stays exact"""
    tile_ids = np.tile(np.arange(3, dtype=np.uint32), 4)
    tile = np.array([2**31 - 1, -2**31, 2**31 - 2, -2**31 + 1, 2**31 - 1, -2**31 + 5,
                     2**31 - 9, -2**31, 7, -2**31 + 3, 2**31 - 1, -1], dtype=np.int32)
    reps = (1 << 28) // len(tile)
    ids = dev(pa.array(np.tile(tile_ids, reps)), ctx)
    vals = dev(pa.array(np.tile(tile, reps)), ctx)
    for fn in ("variance", "stddev"):
        a, b = (bc.HashAggregator("hash_" + fn, pa.int32(), ctx=ctx, ddof=1) for _ in range(2))
        a.resize(3)
        b.resize(3)
        for _ in range(17):
            a.consume(vals, ids)
        b.consume(vals, ids)
        a.merge(b, dev(pa.array(np.arange(3, dtype=np.uint32)), ctx))
        got = a.finalize().to_arrow().to_pylist()
        for g in range(3):
            xs = [int(v) for v in tile[tile_ids == g]]
            k = 18 * reps
            n, s1, s2 = k * len(xs), k * sum(xs), k * sum(v * v for v in xs)
            assert n > 2**30 and s2 > 2**90
            want = float(mr.Fraction(n * s2 - s1 * s1, n * (n - 1)))
            assert got[g] == (math.sqrt(want) if fn == "stddev" else want), (fn, g)


TWO_PASS = [pa.float32(), pa.float64(), pa.int64(), pa.uint64()]


def two_pass_values(t, n, rng):
    """mean 1e3 and spread 1 (condition number about 1e3) for floats; integers offset by 1e12 with spread 1e4"""
    if pa.types.is_floating(t):
        return rng.normal(1e3, 1.0, n).astype(t.to_pandas_dtype())
    return (10**12 + rng.integers(-10**4, 10**4, n)).astype(t.to_pandas_dtype())


@pytest.mark.parametrize("regime", ["private", "atomic", "banded", "merge", "ungrouped"])
@pytest.mark.parametrize("t", TWO_PASS, ids=str)
def test_two_pass_within_data_bound(ctx, t, regime):
    groups, n = {"private": (200, 60_000), "atomic": (3000, 90_000), "banded": REGIMES["banded"], "merge": (3000, 90_000),
                 "ungrouped": (1, 20_000)}[regime]
    rng = np.random.default_rng(SEED + groups + TWO_PASS.index(t))
    ids = rng.integers(0, groups, n).astype(np.uint32)
    raw = two_pass_values(t, n, rng)
    vals = pa.array(raw, t)
    order = np.argsort(ids, kind="stable")
    starts = np.searchsorted(ids[order], np.arange(groups + 1))
    check = range(groups) if groups == 1 else rng.choice(groups, 30, replace=False)
    table = pa.table({"k": ids, "v": vals})
    for fn in ("variance", "stddev", "skew", "kurtosis"):
        for biased in ((True,) if fn in ("variance", "stddev") else (True, False)):
            opts = {} if fn in ("variance", "stddev") else {"biased": biased}
            if regime == "ungrouped":
                got = [getattr(bc, fn)(dev(vals, ctx), **opts).as_py()]
                ref = [getattr(pc, fn)(vals, **opts).as_py()]
            else:
                got = run(ctx, "hash_" + fn, vals, ids, groups, merged=regime == "merge", **opts).to_pylist()
                po = pc.VarianceOptions() if fn in ("variance", "stddev") else pc.SkewOptions(biased=biased)
                res = table.group_by("k", use_threads=False).aggregate([("v", fn, po)])
                ref = dict(zip(res["k"].to_pylist(), res[f"v_{fn}"].to_pylist()))
            for g in check:
                xs = raw[order[starts[g]:starts[g + 1]]]
                if len(np.unique(xs)) < 2 or (not biased and len(xs) < 4):
                    # no spread (0 / NaN) or too few rows for the unbiased form (null): the reference decides
                    assert (got[g] is None and ref[g] is None) or np.float64(got[g]).tobytes() == np.float64(ref[g]).tobytes() \
                        or (ref[g] is not None and got[g] is not None and abs(got[g] - ref[g]) <= 1e-12 * abs(ref[g])), (fn, int(g))
                    continue
                exact = mr.exact_statistic(fn, xs, 0, biased)
                # the relative bound; its absolute form only where the relative one is undefined (a statistic or moment of 0)
                rel = mr.tolerance(fn, xs)
                tol = rel * abs(exact) if exact != 0 and math.isfinite(rel) else mr.tolerance_abs(fn, xs)
                assert abs(got[g] - exact) <= tol, (fn, t, regime, biased, int(g), got[g], exact, tol)
                assert abs(ref[g] - exact) <= tol, (fn, t, "pyarrow", biased, int(g), ref[g], exact, tol)


def group_bounds(vals, ids, groups):
    """per group over its finite valid values: n, m2 and, for k = 2..4, the two-pass rounding bound of sum((x - mu)^k):
    n * 2^-53 * (sum|d|^k + k * (|mu| + max|d|) * sum|d|^(k-1))"""
    ok = np.asarray(vals.is_valid().to_numpy(zero_copy_only=False), bool)
    x = np.asarray(vals.to_numpy(zero_copy_only=False), np.float64)
    ok &= np.isfinite(x)
    x = np.where(ok, x, 0.0)
    n = np.bincount(ids, weights=ok, minlength=groups)
    mu = np.bincount(ids, weights=x, minlength=groups) / np.maximum(n, 1)
    d = np.where(ok, np.abs(x - mu[ids]), 0.0)
    dmax = np.zeros(groups)
    np.maximum.at(dmax, ids, d)
    m2 = np.bincount(ids, weights=d * d, minlength=groups)
    err = {k: n * 2.0 ** -53 * (np.bincount(ids, weights=d ** k, minlength=groups)
                                + k * (np.abs(mu) + dmax) * np.bincount(ids, weights=d ** (k - 1), minlength=groups))
           for k in (2, 3, 4)}
    return n, m2, err


def special_bound(fn, bounds, g):
    """absolute error bound of the statistic from the moment bounds (first order)"""
    n, m2, err = bounds[0][g], bounds[1][g], {k: v[g] for k, v in bounds[2].items()}
    if m2 == 0:
        return 0.0
    if fn in ("variance", "stddev"):
        return 8 * err[2] / max(n - 2, 1)
    # skew ~ sqrt(n) m3 / m2^1.5, kurtosis ~ n m4 / m2^2 (+ the m2 error carried through); unbiased factors are O(1)
    k = 3 if fn == "skew" else 4
    return 64 * n * (err[k] + err[2] * n ** 0.5) / m2 ** (k / 2) * n ** 0.5


@pytest.mark.parametrize("regime", ["private", "atomic"])
@pytest.mark.parametrize("t", [pa.float32(), pa.float64()], ids=str)
def test_special_floats(ctx, t, regime):
    groups, n = REGIMES[regime]
    ids, raw = er.special_float_groups(t.to_pandas_dtype(), groups, n, SEED + groups)
    vals = raw if isinstance(raw, pa.Array) else pa.array(raw, t)
    table = pa.table({"k": ids, "v": vals})
    bounds = group_bounds(vals, ids, groups)
    for fn in ("variance", "stddev", "skew", "kurtosis"):
        for skip_nulls, min_count in ((True, 0), (False, 0), (True, 3)):
            po = (pc.VarianceOptions(skip_nulls=skip_nulls, min_count=min_count) if fn in ("variance", "stddev")
                  else pc.SkewOptions(skip_nulls=skip_nulls, min_count=min_count))
            res = table.group_by("k", use_threads=False).aggregate([("v", fn, po)])
            want = dict(zip(res["k"].to_pylist(), res[f"v_{fn}"].to_pylist()))
            got = run(ctx, "hash_" + fn, vals, ids, groups, skip_nulls=skip_nulls, min_count=min_count).to_pylist()
            for g in range(groups):
                w, x = want[g], got[g]
                if w is None or x is None or math.isnan(w):
                    assert (x is None and w is None) or (x is not None and w is not None and math.isnan(x)), (fn, g, x, w)
                else:
                    assert abs(x - w) <= 2 * special_bound(fn, bounds, g) + 1e-12 * abs(w), (fn, g, x, w)


def test_ungrouped_reproducible(ctx):
    rng = np.random.default_rng(SEED)
    a = pa.array(rng.normal(5.0, 3.0, 3_000_001), mask=rng.random(3_000_001) < 0.01)
    d = dev(a, ctx)
    halves = [dev(a.slice(0, 1_234_567), ctx), dev(a.slice(1_234_567), ctx)]
    for fn in ("variance", "stddev", "skew", "kurtosis"):
        first, second = getattr(bc, fn)(d).as_py(), getattr(bc, fn)(d).as_py()
        assert np.float64(first).tobytes() == np.float64(second).tobytes(), fn
        split = getattr(bc, fn)(halves).as_py()
        assert split == pytest.approx(first, rel=1e-12), fn
        assert getattr(bc, fn)(halves).as_py() == split
        assert first == pytest.approx(getattr(pc, fn)(a).as_py(), rel=1e-12), fn


def test_call_function_options(ctx):
    a = pa.array([1, 2, 3, 4, 100, None], pa.int32())
    d = dev(a, ctx)
    for name, opts in (("variance", pc.VarianceOptions(ddof=1)), ("stddev", pc.VarianceOptions(ddof=2, min_count=9)),
                       ("skew", pc.SkewOptions(biased=False)), ("kurtosis", pc.SkewOptions(skip_nulls=False))):
        got = bc.call_function(name, [d], opts)
        want = pc.call_function(name, [a], opts)
        assert (got.as_py() is None) == (want.as_py() is None), name
        if want.as_py() is not None:
            assert got.as_py() == pytest.approx(want.as_py(), rel=1e-12), name


def test_repeated_merge_destination_is_refused(ctx):
    a, b = (bc.HashAggregator("hash_kurtosis", pa.float64(), ctx=ctx) for _ in range(2))
    a.resize(2)
    b.resize(2)
    with pytest.raises(pa.ArrowInvalid):
        a.merge(b, dev(pa.array([1, 1], pa.uint32()), ctx))


@pytest.mark.parametrize("fn,t", [("hash_variance", pa.int32()), ("hash_skew", pa.float64())])
def test_mapping_beyond_the_state_is_refused(ctx, fn, t):
    a, b = (bc.HashAggregator(fn, t, ctx=ctx) for _ in range(2))
    a.resize(2)
    b.resize(2)
    with pytest.raises(pa.ArrowInvalid):
        a.merge(b, dev(pa.array([0, 2], pa.uint32()), ctx))


def test_negative_ddof_is_refused(ctx):
    d = dev(pa.array([1.0, 2.0, 4.0]), ctx)
    with pytest.raises(pa.ArrowInvalid):
        bc.call_function("variance", [d], pc.VarianceOptions(ddof=-1))


def test_ids_required_for_more_than_one_group(ctx):
    agg = bc.HashAggregator("hash_variance", pa.float64(), ctx=ctx)
    agg.resize(2)
    with pytest.raises(pa.ArrowInvalid):
        agg.consume(dev(pa.array([1.0, 2.0]), ctx), None)
    s = bc.HashAggregator("hash_sum", pa.float64(), ctx=ctx)
    s.resize(1)
    with pytest.raises(pa.ArrowInvalid):
        s.consume(dev(pa.array([1.0, 2.0]), ctx), None)
