"""The fold items in the queue of the folded gather (take_partitioned.cu, "fold under the gather"): the pass that gathers
from the folded float32 table also builds it, each fold group a step ahead of the chunks that read it.

The queue arithmetic of part_sched_kernel and part_fold_gather_kernel is restated here in numpy and checked without a
device: every ticket is one item, every item has one ticket, and no gather chunk reads a fold group whose fold items
do not all have smaller tickets.  On the device the call is compared bit for bit with the direct kernels
(B2_TAKE_PARTITION=0) on index columns that stress the order of the queue."""
import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray

from .util import SEED

TILE = 4096
BUCKETS = 256
FOLD_LEAD = 2  # kFoldLead


def _band_shift(vlen, band_bytes):
    shift = 0
    while (4 << (shift + 1)) <= band_bytes:
        shift += 1
    while ((vlen - 1) >> shift) >= BUCKETS:
        shift += 1
    return shift


def _fold_through(g, group_shift, n_items):
    """fold items in groups 0 .. g (fold_items_through)"""
    return np.minimum((np.asarray(g, np.int64) + 1) << (group_shift - 12), n_items)


def _queue(vlen, shift, n, bucket_start):
    """The queue as the device builds it.  bucket_start[b]: rows of bucket order before bucket b, b = 0 .. 256.
    Returns per ticket (is_fold, item), the step of each ticket (-1: the lead), group_shift and the group count."""
    group_shift = max(shift, 12)
    n_groups = (vlen + (1 << group_shift) - 1) >> group_shift
    n_items = (vlen + TILE - 1) // TILE
    n_tiles = (n + TILE - 1) // TILE
    assert n_groups <= BUCKETS
    # part_sched_kernel
    b = (np.arange(BUCKETS) + 1) << (group_shift - shift)
    p = np.where(b < BUCKETS, bucket_start[np.minimum(b, BUCKETS)], n)
    gather_end = np.where(p == n, n_tiles, p // TILE)
    gather_begin = np.concatenate([[0], gather_end[:-1]])
    # part_fold_gather_kernel
    last = n_groups - 1
    t = np.arange(n_items + n_tiles, dtype=np.int64)
    g = np.arange(n_groups)
    begins = _fold_through(np.minimum(g + FOLD_LEAD - 1, last), group_shift, n_items) + gather_begin[:n_groups]
    assert (np.diff(begins) >= 0).all()
    step = np.searchsorted(begins, t, side="right") - 1
    s = np.maximum(step, 0)
    f0 = _fold_through(np.minimum(s + FOLD_LEAD - 1, last), group_shift, n_items)
    nf = _fold_through(np.minimum(s + FOLD_LEAD, last), group_shift, n_items) - f0
    ng = np.where(s < last, gather_begin[np.minimum(s + 1, BUCKETS - 1)], n_tiles) - gather_begin[s]
    r = t - f0 - gather_begin[s]
    m = np.maximum(nf + ng, 1)
    before = r * nf // m
    is_fold = np.where(step < 0, True, (r + 1) * nf // m > before)
    item = np.where(step < 0, t, np.where(is_fold, f0 + before, gather_begin[s] + r - before))
    return is_fold, item, step, group_shift, n_groups, n_items, n_tiles


def _check_queue(vlen, shift, n, bucket_start, first_bucket=None):
    is_fold, item, step, group_shift, n_groups, n_items, n_tiles = _queue(vlen, shift, n, bucket_start)
    # every ticket is one item and every item has one ticket
    assert sorted(item[is_fold]) == list(range(n_items))
    assert sorted(item[~is_fold]) == list(range(n_tiles))
    # the ticket after which each group is folded: one past the largest ticket among its fold items
    fold_ticket = np.flatnonzero(is_fold)
    fold_group = (item[is_fold] * TILE) >> group_shift
    folded_at = np.zeros(n_groups, np.int64)
    np.maximum.at(folded_at, fold_group, fold_ticket + 1)
    assert (np.bincount(fold_group, minlength=n_groups) > 0).all()
    ready = np.maximum.accumulate(folded_at)  # all groups <= g are folded from this ticket on
    # a chunk reads the groups of its first to its last position; the last is its step, which the kernel waits up to
    chunk_ticket = np.flatnonzero(~is_fold)
    chunk = item[~is_fold]
    last_pos = np.minimum(chunk * TILE + TILE - 1, n - 1)
    last_bucket = np.searchsorted(bucket_start[1:], last_pos, side="right")
    last_group = (last_bucket << shift) >> group_shift
    assert np.array_equal(last_group, step[~is_fold])
    assert (ready[last_group] <= chunk_ticket).all()


def _bucket_start(buckets, n):
    return np.concatenate([np.searchsorted(np.sort(buckets), np.arange(BUCKETS)), [n]])


QUEUE_SHAPES = [  # (values_length, n, band bytes of the folded table): the first six are test_gpu_take_fold.py's CASES
    (70001, 200003, 4 << 10), (70001, 200003, 4 << 10), (5000, 4097, 1 << 10), (9999, 30000, 64 << 10),
    (70001, 200003, 4 << 10), (12289, 50000, 16 << 10),
    (600_000, 1_000_000, 64 << 10),     # several fold items per band, many bands
    ((1 << 14) + 1, 50_000, 64 << 10),  # one band and one row
    (4096 * 7 + 5, 4096 * 3, 16 << 10),
    (1000, 8192, 1 << 10),              # fewer values than one fold item
]


@pytest.mark.parametrize("shape", range(len(QUEUE_SHAPES)))
@pytest.mark.parametrize("pattern", ["uniform", "one_band", "last_band", "empty_bands"])
def test_queue_is_a_permutation_and_ordered(shape, pattern):
    vlen, n, band = QUEUE_SHAPES[shape]
    rng = np.random.default_rng(SEED + shape)
    shift = _band_shift(vlen, band)
    j = rng.integers(0, vlen, n)
    if pattern == "one_band":
        j = j % min(vlen, 1 << shift)
    elif pattern == "last_band":
        j = np.maximum(j, ((vlen - 1) >> shift) << shift)
    elif pattern == "empty_bands":
        j = np.where(((j >> shift) % 3) == 1, j, j % min(vlen, 1 << shift))
    _check_queue(vlen, shift, n, _bucket_start(j >> shift, n))


def test_queue_at_the_bench_shape():
    """1e9 float64 values, 1e9 uniform rows, 16 MB bands of the folded table: bucket starts at their expectation"""
    vlen = n = 1_000_000_000
    shift = _band_shift(vlen, 16 << 20)
    assert shift == 22
    edges = np.minimum(np.arange(BUCKETS + 1, dtype=np.int64) << shift, vlen)
    _check_queue(vlen, shift, n, edges * n // vlen)


# ---- on the device ---------------------------------------------------------------------------------------------------
def _values(vlen, rng):
    data = rng.uniform(-1e6, 1e6, vlen)
    data[::11] = np.nan
    return pa.array(data, pa.float64(), mask=rng.random(vlen) < 0.1)


def _run(monkeypatch, partition, band_kb, fn):
    monkeypatch.setenv("B2_TAKE_PARTITION", partition)
    if partition == "1":
        monkeypatch.setenv("B2_TAKE_PART_BAND_KB", str(band_kb))
    else:
        monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
    return fn().to_arrow()


def _same_bits(a, b):
    assert len(a) == len(b) and a.null_count == b.null_count
    assert a.buffers()[1].to_pybytes()[a.offset * 4:(a.offset + len(a)) * 4] == \
        b.buffers()[1].to_pybytes()[b.offset * 4:(b.offset + len(b)) * 4]
    va = np.asarray(a.is_valid())
    assert np.array_equal(va, np.asarray(b.is_valid()))


def _check(ctx, monkeypatch, vlen, raw, band_kb, seed):
    rng = np.random.default_rng(SEED + seed)
    n = len(raw)
    values = _values(vlen, rng)
    idx = pa.array(raw, pa.int64(), mask=rng.random(n) < 0.05)
    other = pa.array(rng.uniform(-10, 10, n).astype(np.float32), pa.float32(), mask=rng.random(n) < 0.1)
    dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, other))
    fn = lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do)  # noqa: E731
    _same_bits(_run(monkeypatch, "1", band_kb, fn), _run(monkeypatch, "0", band_kb, fn))


@pytest.mark.gpu
def test_all_rows_in_the_last_band(ctx, monkeypatch):
    """every chunk waits on the fold items that come last"""
    rng = np.random.default_rng(SEED)
    vlen, band_rows = 600_000, 16384
    lo = ((vlen - 1) // band_rows) * band_rows
    _check(ctx, monkeypatch, vlen, rng.integers(lo, vlen, 300_000), 64, 1)


@pytest.mark.gpu
def test_rows_in_descending_band_order(ctx, monkeypatch):
    rng = np.random.default_rng(SEED + 1)
    vlen = 600_000
    raw = rng.integers(0, vlen, 500_000)
    raw = raw[np.argsort(-(raw // 16384), kind="stable")]
    _check(ctx, monkeypatch, vlen, raw, 64, 2)


@pytest.mark.gpu
def test_many_bands_of_several_fold_items(ctx, monkeypatch):
    """37 bands of four fold items each under a million rows: the steady part of the queue"""
    rng = np.random.default_rng(SEED + 2)
    _check(ctx, monkeypatch, 600_000, rng.integers(0, 600_000, 1_000_000), 64, 3)


@pytest.mark.gpu
def test_chunk_straddling_three_buckets(ctx, monkeypatch):
    """4000 rows in band 0, 50 in band 5, the rest in band 9: chunk 0 reads all three"""
    rng = np.random.default_rng(SEED + 3)
    vlen, band_rows = 600_000, 16384
    raw = np.concatenate([rng.integers(0, band_rows, 4000), rng.integers(5 * band_rows, 6 * band_rows, 50),
                          rng.integers(9 * band_rows, 10 * band_rows, 20_000)])
    _check(ctx, monkeypatch, vlen, rng.permutation(raw), 64, 4)


@pytest.mark.gpu
def test_one_band_and_one_row(ctx, monkeypatch):
    rng = np.random.default_rng(SEED + 4)
    vlen = 16384 + 1
    raw = rng.integers(0, vlen, 100_000)
    raw[::100] = vlen - 1
    _check(ctx, monkeypatch, vlen, raw, 64, 5)


@pytest.mark.gpu
def test_the_fold_runs_inside_the_gather_launch(ctx, monkeypatch):
    """one launch folds and gathers; no stand-alone fold kernel is left"""
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(SEED + 5)
    vlen, n = 200_000, 300_000
    dv = DeviceArray.from_arrow(_values(vlen, rng), ctx)
    di = DeviceArray.from_arrow(pa.array(rng.integers(0, vlen, n), pa.int64()), ctx)
    do = DeviceArray.from_arrow(pa.array(rng.uniform(-1, 1, n).astype(np.float32)), ctx)
    fn = lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do)  # noqa: E731
    _run(monkeypatch, "1", 64, fn)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run(monkeypatch, "1", 64, fn)
    names = [e.key for e in prof.key_averages()]
    assert any("part_fold_gather_kernel" in k for k in names), names
    assert not any("fold_kernel<" in k or "part_gather_kernel" in k for k in names), names
