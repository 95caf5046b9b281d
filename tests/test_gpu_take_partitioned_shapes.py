"""The partitioned path of b2_take / b2_take_cast_arith on index distributions the random cases of
test_gpu_take_partitioned.py do not reach: one bucket spanning many 4096-position chunks, long stretches of empty
(tile, bucket) cells, no valid index at all, and a partial last tile that falls entirely in the last bucket.  Forced with
B2_TAKE_PARTITION=1 and 1 KB bands, and compared bit for bit with the direct kernels (B2_TAKE_PARTITION=0)."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from oracle import arrow_oracle as ora

from .test_gpu_take_partitioned import _run, _same_bits
from .util import SEED

pytestmark = pytest.mark.gpu

TILE = 4096
N_VALUES = 256 * 128  # float64 values in 1 KB bands: 128 rows per bucket, exactly 256 buckets


def _one_bucket(rng):
    """hundreds of whole tiles in bucket 100: that bucket spans ~300 chunks and every tile's count is 4096"""
    n = 300 * TILE + 123
    return rng.integers(100 * 128, 101 * 128, n), None


def _sparse_far_buckets(rng):
    """everything in bucket 0 except a handful of rows in distant buckets: long columns of empty cells"""
    n = 200 * TILE + 7
    raw = rng.integers(0, 128, n)
    for row, bucket in ((5, 255), (77_777, 128), (400_000, 255), (n - 1, 200), (n - 2, 1)):
        raw[row] = bucket * 128 + 3
    return raw, None


def _all_null(rng):
    n = 50 * TILE + 1000
    return rng.integers(0, N_VALUES, n), np.ones(n, bool)


def _last_tile_in_last_bucket(rng):
    """the partial last tile's rows all fall in bucket 255; the whole tiles before it are uniform"""
    n = 20 * TILE + 1000
    raw = rng.integers(0, N_VALUES, n)
    raw[20 * TILE:] = rng.integers(255 * 128, N_VALUES, 1000)
    return raw, rng.random(n) < 0.05


SHAPES = [_one_bucket, _sparse_far_buckets, _all_null, _last_tile_in_last_bucket]


@pytest.mark.parametrize("it", [pa.int32(), pa.int64()], ids=str)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda f: f.__name__.lstrip("_"))
def test_partitioned_skewed_shapes_equal_direct(ctx, monkeypatch, shape, it):
    rng = np.random.default_rng(SEED)
    values = pa.array(rng.uniform(-1e6, 1e6, N_VALUES), pa.float64(), mask=rng.random(N_VALUES) < 0.1)
    raw, mask = shape(rng)
    n = len(raw)
    idx = pa.array(raw, it, mask=mask)
    other = pa.array(rng.uniform(-10, 10, n).astype(np.float32), pa.float32(), mask=rng.random(n) < 0.1)
    dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, other))

    part = _run(monkeypatch, "1", 1, lambda: bc.take(dv, di))
    direct = _run(monkeypatch, "0", 1, lambda: bc.take(dv, di))
    _same_bits(part, direct)
    assert part.equals(ora.take(values, idx))

    part = _run(monkeypatch, "1", 1, lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do))
    direct = _run(monkeypatch, "0", 1, lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do))
    _same_bits(part, direct)
    want = pc.add(pc.cast(pc.take(values, idx), pa.float32(), safe=False), other)
    assert part.equals(want) and part.null_count == want.null_count
