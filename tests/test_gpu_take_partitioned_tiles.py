"""The partitioned path of b2_take / b2_take_cast_arith around its 4096-row partition tiles and 4096-position gather
chunks: row counts at the tile edges, runs of a whole tile that start inside a chunk or on its first position, runs
that start or end at a chunk boundary, a partial last tile in the last bucket, long stretches of empty cells, no valid
index, and the first out-of-range index in the second half of a tile.  Forced with B2_TAKE_PARTITION=1 and KB bands,
and compared bit for bit with the direct kernels (B2_TAKE_PARTITION=0): every value slot, null or not, every validity
bit, the null count and the IndexError.  Each case runs a plain take of 4- and 8-byte values and a take + cast + add to float32 with and without
the folded gather.

Bands are 256 rows in every call (1 KB of float32 / of the folded table, 2 KB of float64) over 65536 values, so the
bucket of index j is j >> 8 for all four calls."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi

from .util import SEED

pytestmark = pytest.mark.gpu

TILE = 4096   # rows of a partition tile (passes A and C)
CHUNK = 4096  # positions of a gather chunk (pass B)
BUCKET_ROWS = 256
N_VALUES = 256 * BUCKET_ROWS
FOLD_LAUNCHES = 3  # count, scan, sched: the folded call's launches beyond the unfolded one's


def _in_buckets(rng, buckets, n):
    """n indices, each in a bucket drawn from `buckets`"""
    return np.asarray(buckets)[rng.integers(0, len(buckets), n)] * BUCKET_ROWS + rng.integers(0, BUCKET_ROWS, n)


def _call(monkeypatch, partition, band_kb, fn):
    monkeypatch.setenv("B2_TAKE_PARTITION", partition)
    if partition == "1":
        monkeypatch.setenv("B2_TAKE_PART_BAND_KB", str(band_kb))
    else:
        monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
    lib = _cabi.lib()
    before = lib.b2_launch_count()
    out = fn().to_arrow()
    return out, lib.b2_launch_count() - before


def _same_bits(a, b):
    """every slot's bytes, null or not, and every validity bit"""
    assert len(a) == len(b) and a.type == b.type and a.null_count == b.null_count
    w = a.type.bit_width // 8
    assert a.buffers()[1].to_pybytes()[a.offset * w:(a.offset + len(a)) * w] == \
        b.buffers()[1].to_pybytes()[b.offset * w:(b.offset + len(b)) * w]
    if a.null_count:
        va = np.unpackbits(np.frombuffer(a.buffers()[0], np.uint8), bitorder="little")[a.offset:a.offset + len(a)]
        vb = np.unpackbits(np.frombuffer(b.buffers()[0], np.uint8), bitorder="little")[b.offset:b.offset + len(b)]
        assert np.array_equal(va, vb)


def _calls(ctx, rng, idx):
    """(name, band KB, fn) for the four calls over `idx`, and the float64 and float32 values they read"""
    n = len(idx)
    v64 = pa.array(rng.uniform(-1e6, 1e6, N_VALUES), pa.float64(), mask=rng.random(N_VALUES) < 0.1)
    v32 = pa.array(rng.uniform(-1e6, 1e6, N_VALUES).astype(np.float32), pa.float32(), mask=rng.random(N_VALUES) < 0.1)
    o32 = pa.array(rng.uniform(-10, 10, n).astype(np.float32), pa.float32(), mask=rng.random(n) < 0.1)
    dv64, dv32, di, do32 = (DeviceArray.from_arrow(x, ctx) for x in (v64, v32, idx, o32))
    do64 = DeviceArray.from_arrow(o32.cast(pa.float64()), ctx)
    return [
        ("take float32", 1, lambda: bc.take(dv32, di)),
        ("take float64", 2, lambda: bc.take(dv64, di)),
        ("take_cast_arith float64 -> float32, folded", 1, lambda: bc.take_cast_arith(dv64, di, pa.float32(), "add", do32)),
        ("take_cast_arith float64 -> float64", 2, lambda: bc.take_cast_arith(dv64, di, pa.float64(), "add", do64)),
    ], (v64, v32)


def _check(ctx, monkeypatch, raw, mask=None, it=pa.int64(), seed=0):
    rng = np.random.default_rng(SEED + seed)
    idx = pa.array(raw, it, mask=mask)
    calls, _ = _calls(ctx, rng, idx)
    launches = {}
    for name, band_kb, fn in calls:
        part, launches[name] = _call(monkeypatch, "1", band_kb, fn)
        direct, _ = _call(monkeypatch, "0", band_kb, fn)
        _same_bits(part, direct)
    assert launches[calls[2][0]] - launches[calls[3][0]] == FOLD_LAUNCHES  # the float32 call took the folded gather


# ---- row counts at the tile edges ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4095, 4096, 4097, 8191, 8192, 8193, 16383, 16385])
def test_tile_edges(ctx, monkeypatch, n):
    rng = np.random.default_rng(SEED + n)
    _check(ctx, monkeypatch, rng.integers(0, N_VALUES, n), rng.random(n) < 0.05, pa.int32() if n & 1 else pa.int64(), n)


# ---- run shapes ------------------------------------------------------------------------------------------------------
def _last_tile_in_last_bucket(rng):
    """uniform whole tiles, then a partial last tile entirely in bucket 255 (with the tile's padding, also bucket 255)"""
    n = 10 * TILE + 1000
    raw = rng.integers(0, N_VALUES, n)
    raw[10 * TILE:] = _in_buckets(rng, [255], 1000)
    return raw, rng.random(n) < 0.05


def _whole_tiles_in_one_bucket(rng):
    """the first two tiles put 1000 rows in bucket 0 and 3000 in bucket 200, so bucket 100 starts at position 1000 of
    bucket order; every later tile lies wholly in bucket 100, and each of its runs holds a chunk start that is not its
    first position"""
    n = 18 * TILE + 4321
    raw = _in_buckets(rng, [100], n)
    head = np.concatenate([_in_buckets(rng, [0], 1000), _in_buckets(rng, [200], 3000),
                           _in_buckets(rng, [100], 2 * TILE - 4000)])
    raw[:2 * TILE] = rng.permutation(head)
    return raw, None


def _whole_tiles_chunk_aligned(rng):
    """every tile wholly in bucket 77: each run is exactly one chunk"""
    n = 12 * TILE
    return _in_buckets(rng, [77], n), rng.random(n) < 0.02


def _runs_at_a_chunk_boundary(rng):
    """bucket 3 holds 4095 rows of tile 0 and 1 row of tile 1: tile 1's run starts at position 4095, one before the
    chunk boundary, and ends exactly on it; tile 0's one row of bucket 7 then starts a run exactly on the boundary"""
    n = 6 * TILE + 5
    t0 = np.concatenate([_in_buckets(rng, [3], CHUNK - 1), _in_buckets(rng, [7], TILE - CHUNK + 1)])
    rest = _in_buckets(rng, np.arange(8, 256), n - TILE)
    rest[rng.integers(0, TILE)] = _in_buckets(rng, [3], 1)[0]  # tile 1's single row of bucket 3
    return np.concatenate([rng.permutation(t0), rest]), None


def _sparse_far_buckets(rng):
    """everything in bucket 0 but a handful of rows in distant buckets: long columns of empty cells, and runs of
    bucket 0 that are whole tiles"""
    n = 80 * TILE + 7
    raw = _in_buckets(rng, [0], n)
    for row, bucket in ((5, 255), (TILE + 4000, 128), (35 * TILE + 3000, 255), (n - 1, 200), (n - 2, 1)):
        raw[row] = bucket * BUCKET_ROWS + 3
    return raw, None


def _all_null(rng):
    n = 20 * TILE + 1000
    return rng.integers(0, N_VALUES, n), np.ones(n, bool)


SHAPES = [_last_tile_in_last_bucket, _whole_tiles_in_one_bucket, _whole_tiles_chunk_aligned, _runs_at_a_chunk_boundary,
          _sparse_far_buckets, _all_null]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda f: f.__name__.lstrip("_"))
def test_run_shapes(ctx, monkeypatch, shape):
    rng = np.random.default_rng(SEED)
    raw, mask = shape(rng)
    _check(ctx, monkeypatch, raw, mask)


# ---- index errors ----------------------------------------------------------------------------------------------------
def test_first_bad_index_in_second_half_of_a_tile(ctx, monkeypatch):
    """out-of-range indices in the second half of tile 1 (the lowest is named) and in tile 2; a null one below them
    is never checked"""
    rng = np.random.default_rng(SEED + 7)
    n = 3 * TILE + 100
    raw = rng.integers(0, N_VALUES, n)
    mask = np.zeros(n, bool)
    raw[TILE + 3500], raw[TILE + 3000], raw[2 * TILE + 10] = N_VALUES + 1, N_VALUES, N_VALUES + 1000
    raw[TILE + 100], mask[TILE + 100] = N_VALUES + 5, True
    idx = pa.array(raw, pa.int64(), mask=mask)
    calls, (v64, _) = _calls(ctx, rng, idx)
    with pytest.raises(pa.ArrowIndexError) as want:
        pc.take(v64, idx)
    assert str(want.value) == f"Index {N_VALUES} out of bounds"  # row TILE + 3000's
    for name, band_kb, fn in calls:
        msgs = []
        for partition in ("1", "0"):
            with pytest.raises(pa.ArrowIndexError) as err:
                _call(monkeypatch, partition, band_kb, fn)
            msgs.append(str(err.value))
        assert msgs[0] == msgs[1] == str(want.value), name
