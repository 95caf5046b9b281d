"""The numpy restatement of variance / stddev / skew / kurtosis (tests/moments_ref.py) pinned against pyarrow, and the
exact Fraction helpers against it.  CPU only."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import moments_ref as mr
from tests.util import SEED

TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64(),
         pa.float32(), pa.float64()]
FUNCS = ["variance", "stddev", "skew", "kurtosis"]


def _values(t, n, rng, nulls=0.1):
    if pa.types.is_floating(t):
        v = rng.normal(3.0, 2.0, n).astype(t.to_pandas_dtype())
    else:
        info = np.iinfo(t.to_pandas_dtype())
        lo, hi = max(int(info.min), -1000), min(int(info.max), 1000)
        v = rng.integers(lo, hi + 1, n).astype(t.to_pandas_dtype())
    return pa.array(v, t, mask=rng.random(n) < nulls)


def _close(got, want, rtol=1e-9):
    if want is None or got is None:
        return got is None and want is None
    if math.isnan(want):
        return math.isnan(got)
    return got == pytest.approx(want, rel=rtol, abs=1e-300)


def _opts(fn, ddof, biased, skip_nulls, min_count):
    if fn in ("variance", "stddev"):
        return pc.VarianceOptions(ddof=ddof, skip_nulls=skip_nulls, min_count=min_count), dict(ddof=ddof)
    return pc.SkewOptions(skip_nulls=skip_nulls, biased=biased, min_count=min_count), dict(biased=biased)


@pytest.mark.parametrize("t", TYPES, ids=str)
@pytest.mark.parametrize("fn", FUNCS)
def test_scalar_matches_pyarrow(t, fn):
    rng = np.random.default_rng(SEED + 16 * TYPES.index(t) + FUNCS.index(fn))
    chunks = [_values(t, n, rng) for n in (0, 37, 200, 5)]
    ca = pa.chunked_array(chunks, t)
    for ddof, biased in ((0, True), (1, False), (2, True)):
        for skip_nulls in (True, False):
            for min_count in (0, 1, 5):
                po, extra = _opts(fn, ddof, biased, skip_nulls, min_count)
                want = getattr(pc, fn)(ca, options=po).as_py()
                got = mr.scalar(fn, chunks, skip_nulls=skip_nulls, min_count=min_count, **extra)
                assert _close(got, want), (fn, t, ddof, biased, skip_nulls, min_count, got, want)


@pytest.mark.parametrize("t", TYPES, ids=str)
@pytest.mark.parametrize("fn", FUNCS)
def test_grouped_matches_pyarrow(t, fn):
    rng = np.random.default_rng(SEED + 1000 + 16 * TYPES.index(t) + FUNCS.index(fn))
    g = 6
    batches = []
    for n in (120, 45):
        batches.append((_values(t, n, rng), rng.integers(0, g, n).astype(np.uint32)))
    # group 5: a handful of rows only, so min_count / ddof / unbiased thresholds bite
    batches[0][1][batches[0][1] == 5] = 4
    batches[1][1][:3] = 5
    batches[1][1][3:][batches[1][1][3:] == 5] = 0
    table = pa.Table.from_batches([pa.record_batch([ids, vals], names=["k", "v"]) for vals, ids in
                                   ((v, pa.array(i)) for v, i in batches)])
    for ddof, biased in ((0, True), (1, False), (2, True)):
        for skip_nulls in (True, False):
            for min_count in (0, 1, 5):
                po, extra = _opts(fn, ddof, biased, skip_nulls, min_count)
                res = table.group_by("k", use_threads=False).aggregate([("v", fn, po)]).sort_by("k")
                want = dict(zip(res["k"].to_pylist(), res[f"v_{fn}"].to_pylist()))
                got = mr.grouped(fn, batches, g, skip_nulls=skip_nulls, min_count=min_count, **extra)
                for k in range(g):
                    assert _close(got[k], want[k]), (fn, t, k, ddof, biased, skip_nulls, min_count, got[k], want[k])


@pytest.mark.parametrize("t", [pa.int8(), pa.uint16(), pa.int32(), pa.uint32()], ids=str)
def test_exact_fraction_helpers(t):
    rng = np.random.default_rng(SEED + 11)
    info = np.iinfo(t.to_pandas_dtype())
    vals = rng.integers(int(info.min), int(info.max), 300, dtype=np.int64, endpoint=True)
    for ddof in (0, 1, 2):
        exact = mr.exact_variance(vals, ddof)
        assert exact == mr.exact_central(vals, 2) / (len(vals) - ddof)
        ora = mr.scalar("variance", [pa.array(vals, t)], ddof=ddof)
        assert ora == pytest.approx(float(exact), rel=4 * 2.0 ** -52)   # the reference rounds twice
        assert mr.exact_statistic("stddev", vals, ddof) == math.sqrt(float(exact))


def test_tolerance_covers_the_oracle():
    rng = np.random.default_rng(SEED + 5)
    vals = rng.normal(100.0, 3.0, 500)
    for fn in FUNCS:
        for biased in (True, False):
            want = mr.exact_statistic(fn, vals, 0, biased)
            got = mr.scalar(fn, [pa.array(vals)], biased=biased)
            assert abs(got - want) <= mr.tolerance(fn, vals) * abs(want), (fn, biased, got, want)
