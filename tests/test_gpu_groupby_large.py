"""The partitioned (hash radix-partition + shared-memory pre-aggregation) path of the fused
group-by, which only engages from 2^21 rows: 0, 1 and 2 partition passes, null keys, null values,
the all-ones key, several consume() batches, and growth past the cardinality hint -- against the
reference engine (Acero via pyarrow, rows sorted by key as its own tests do)."""
import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi

pytestmark = pytest.mark.gpu
SEED = 0x0FF1CE


def reference(keys, vals):
    import pyarrow.acero  # noqa: F401
    t = pa.table({"k": keys, "v": vals}).group_by("k", use_threads=False).aggregate([("v", "sum"), ("v", "count")])
    return t.sort_by("k")


def check(ctx, keys, vals, hint, batches=1):
    g = bc.GroupBySumCount(keys.type, vals.type, expected_groups=hint, ctx=ctx)
    n = len(keys)
    dk, dv = DeviceArray.from_arrow(keys, ctx), DeviceArray.from_arrow(vals, ctx)
    for b in range(batches):
        lo, hi = b * n // batches, (b + 1) * n // batches
        g.consume(dk.slice(lo, hi - lo), dv.slice(lo, hi - lo))
    k, s, c = [x.to_arrow() for x in g.finalize()]
    got = pa.table({"k": k, "v_sum": s, "v_count": c}).sort_by("k")
    want = reference(keys, vals)
    assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
    assert got["v_count"].combine_chunks().equals(want["v_count"].combine_chunks())
    gs, ws = got["v_sum"].combine_chunks(), want["v_sum"].combine_chunks()
    if pa.types.is_integer(vals.type):
        assert gs.equals(ws)
    else:
        assert gs.is_valid().equals(ws.is_valid())
        np.testing.assert_allclose(gs.fill_null(0).to_numpy(), ws.fill_null(0).to_numpy(), rtol=1e-9, atol=1e-6)


@pytest.mark.parametrize("groups,hint", [(100, 100), (50_000, 50_000), (600_000, 600_000), (600_000, 0), (600_000, 1000)])
def test_partitioned_group_by_int64(ctx, groups, hint):
    n = 3_000_000
    rng = np.random.default_rng(SEED + groups)
    k = rng.integers(0, groups, n, dtype=np.int64)
    k[:3] = [-1, np.iinfo(np.int64).min, np.iinfo(np.int64).max]   # 0xFFFF.. is the table's empty marker
    keys = pa.array(k, mask=rng.random(n) < 0.01)
    vals = pa.array(rng.integers(-100, 100, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    check(ctx, keys, vals, hint)


def test_partitioned_group_by_types_and_batches(ctx):
    n = 2_500_000
    rng = np.random.default_rng(SEED)
    keys32 = pa.array(rng.integers(-70000, 70000, n, dtype=np.int32), mask=rng.random(n) < 0.02)
    fvals = pa.array(rng.uniform(-1, 1, n), pa.float64(), mask=rng.random(n) < 0.1)
    check(ctx, keys32, fvals, 140_000)
    u16 = pa.array(rng.integers(0, 60000, n, dtype=np.uint16))
    f32 = pa.array(rng.uniform(0, 10, n).astype(np.float32), mask=rng.random(n) < 0.5)
    check(ctx, u16, f32, 0)
    # a group whose every value is null must exist with sum = null, count = 0
    k = rng.integers(0, 500_000, n, dtype=np.int64)
    v = rng.integers(-5, 5, n, dtype=np.int64)
    mask = (k % 7 == 0) | (rng.random(n) < 0.05)
    check(ctx, pa.array(k), pa.array(v, mask=mask), 500_000)
    # several consume() calls, each above the partitioning threshold; growing past the hint
    k2 = pa.array(rng.integers(0, 900_000, 3 * n, dtype=np.int64))
    v2 = pa.array(rng.integers(-100, 100, 3 * n, dtype=np.int64), mask=rng.random(3 * n) < 0.1)
    check(ctx, k2, v2, 10_000, batches=3)


# ---- the compact path (csrc/groupby_compact.cuh): 8-byte tuples, bulk-async partition passes ----------
def check_path(ctx, keys, vals, hint, want_path, batches=1, offset=0):
    g = bc.GroupBySumCount(keys.type, vals.type, expected_groups=hint, ctx=ctx)
    n = len(keys)
    dk, dv = DeviceArray.from_arrow(keys, ctx), DeviceArray.from_arrow(vals, ctx)
    keys, vals = keys.slice(offset), vals.slice(offset)
    dk, dv = dk.slice(offset), dv.slice(offset)
    n -= offset
    for b in range(batches):
        lo, hi = b * n // batches, (b + 1) * n // batches
        g.consume(dk.slice(lo, hi - lo), dv.slice(lo, hi - lo))
    paths = g.path_counts()
    if want_path is not None:
        assert paths[want_path] == batches and sum(paths.values()) == batches, paths
    k, s, c = [x.to_arrow() for x in g.finalize()]
    got = pa.table({"k": k, "v_sum": s, "v_count": c}).sort_by("k")
    want = reference(keys, vals)
    assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
    assert got["v_count"].combine_chunks().equals(want["v_count"].combine_chunks())
    assert got["v_sum"].combine_chunks().equals(want["v_sum"].combine_chunks())


@pytest.mark.parametrize("groups,hint", [(50_000, 50_000), (600_000, 600_000), (600_000, 0)])
@pytest.mark.parametrize("offset", [0, 1])
def test_compact_group_by_narrow(ctx, groups, hint, offset):
    """int64 keys in [0, groups), int64 values in [-100, 100]: 32-bit shared-memory slots; offset 1 makes the
    column pointers 8- but not 16-byte aligned, which takes the plain-load branch of the tile loader"""
    n = 3_000_001 + offset
    rng = np.random.default_rng(SEED + groups + offset)
    keys = pa.array(rng.integers(0, groups, n, dtype=np.int64), mask=rng.random(n) < 0.01)
    vals = pa.array(rng.integers(-100, 101, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    check_path(ctx, keys, vals, hint, "compact", offset=offset)


def test_compact_group_by_wide_slots_types_and_batches(ctx):
    n = 2_600_000
    rng = np.random.default_rng(SEED + 7)
    # key range 2^40, value range 2^21: 64-bit shared-memory slots
    k = pa.array(rng.integers(-2**39, 2**39, 400_000, dtype=np.int64)[rng.integers(0, 400_000, n)], mask=rng.random(n) < 0.02)
    v = pa.array(rng.integers(-2**20, 2**20, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    check_path(ctx, k, v, 400_000, "compact")
    # narrow native types: the value window is the type's own range (nothing sampled)
    k32 = pa.array(rng.integers(-70000, 70000, n, dtype=np.int32), mask=rng.random(n) < 0.02)
    v16 = pa.array(rng.integers(-30000, 30000, n, dtype=np.int16), mask=rng.random(n) < 0.1)
    check_path(ctx, k32, v16, 140_000, "compact")
    ku16 = pa.array(rng.integers(0, 60000, n, dtype=np.uint16))
    vu8 = pa.array(rng.integers(0, 255, n, dtype=np.uint8), mask=rng.random(n) < 0.5)
    check_path(ctx, ku16, vu8, 0, "compact")
    vu64 = pa.array(rng.integers(2**63, 2**63 + 1000, n, dtype=np.uint64), mask=rng.random(n) < 0.1)  # sums wrap like the reference
    check_path(ctx, ku16, vu64, 60_000, "compact")
    # a group whose every value is null must exist with sum = null, count = 0; an all-null-key batch
    kk = rng.integers(0, 500_000, n, dtype=np.int64)
    vv = rng.integers(-5, 5, n, dtype=np.int64)
    check_path(ctx, pa.array(kk), pa.array(vv, mask=(kk % 7 == 0) | (rng.random(n) < 0.05)), 500_000, "compact")
    check_path(ctx, pa.array(kk, mask=np.ones(n, dtype=bool)), pa.array(vv), 0, None)
    # several consume() calls, growing past the hint
    k2 = pa.array(rng.integers(0, 900_000, 3 * n, dtype=np.int64))
    v2 = pa.array(rng.integers(-100, 100, 3 * n, dtype=np.int64), mask=rng.random(3 * n) < 0.1)
    check_path(ctx, k2, v2, 10_000, "compact", batches=3)


def test_compact_value_window_is_verified_not_trusted(ctx):
    """64-bit values: the window comes from a SAMPLE; one row far outside it (at an unsampled position) must
    send the chunk to the general path, never corrupt the sum"""
    n = 2_500_000
    rng = np.random.default_rng(SEED + 11)
    k = pa.array(rng.integers(0, 300_000, n, dtype=np.int64))
    v = rng.integers(-100, 101, n, dtype=np.int64)
    v[1_234_567] = 2**61 + 12345          # n / 65536 = 38: row 1234567 is not a multiple of 38
    v[1_234_569] = -2**62
    assert 1_234_567 % (n // 65536) != 0 and 1_234_569 % (n // 65536) != 0
    m = rng.random(n) < 0.1
    m[1_234_567] = m[1_234_569] = False
    check_path(ctx, k, pa.array(v, mask=m), 300_000, "general")
    # and the general path on data the compact path would take (B2_GROUPBY_COMPACT=0)
    import os
    os.environ["B2_GROUPBY_COMPACT"] = "0"
    try:
        v2 = pa.array(rng.integers(-100, 101, n, dtype=np.int64), mask=rng.random(n) < 0.1)
        check_path(ctx, k, v2, 300_000, "general")
    finally:
        del os.environ["B2_GROUPBY_COMPACT"]


def test_fused_merge_of_partial_states(ctx):
    """b2_groupby_sumcount_merge: the partial (key, sum, count) tables of two shards added into a third table must
    equal one group-by over all rows (what the owner GPU does after the exchange, and GroupByNode::Merge per thread)"""
    n = 2_400_000
    rng = np.random.default_rng(SEED + 21)
    for vt, mk in ((pa.int64(), lambda: rng.integers(-100, 101, n, dtype=np.int64)), (pa.float64(), lambda: rng.uniform(-1, 1, n)),
                   (pa.uint32(), lambda: rng.integers(0, 1000, n, dtype=np.uint32))):
        keys = pa.array(rng.integers(0, 300_000, n, dtype=np.int64), mask=rng.random(n) < 0.01)
        kk = keys.to_numpy(zero_copy_only=False)
        vals = pa.array(mk(), vt, mask=(rng.random(n) < 0.1) | (np.nan_to_num(kk, nan=1) % 11 == 0))  # some groups: only null values
        parts = []
        for lo, hi in ((0, n // 3), (n // 3, n)):
            g = bc.GroupBySumCount(keys.type, vt, ctx=ctx)
            g.consume(DeviceArray.from_arrow(keys.slice(lo, hi - lo), ctx), DeviceArray.from_arrow(vals.slice(lo, hi - lo), ctx))
            parts.append(g.finalize())
        sum_type = parts[0][1].type
        m = bc.GroupBySumCount(keys.type, sum_type, ctx=ctx)
        for k, s, c in parts:
            m.merge(k, s, c)
        k, s, c = [x.to_arrow() for x in m.finalize()]
        got = pa.table({"k": k, "v_sum": s, "v_count": c}).sort_by("k")
        want = reference(keys, vals)
        assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
        assert got["v_count"].combine_chunks().equals(want["v_count"].combine_chunks())
        gs, ws = got["v_sum"].combine_chunks(), want["v_sum"].combine_chunks()
        if pa.types.is_integer(vt):
            assert gs.equals(ws.cast(gs.type))
        else:
            assert gs.is_valid().equals(ws.is_valid())
            np.testing.assert_allclose(gs.fill_null(0).to_numpy(), ws.fill_null(0).to_numpy(), rtol=1e-9, atol=1e-6)


# ---- the direct-addressed path (csrc/groupby_dense.cuh): dense keys, packed state in L2 -----------------------------
@pytest.mark.parametrize("offset", [0, 1])
def test_dense_group_by(ctx, offset):
    """>= 2^22 rows over a dense key range: one reduction per row into table[key - kmin]"""
    n = 4_700_000 + offset
    rng = np.random.default_rng(SEED + 31 + offset)
    keys = pa.array(rng.integers(-250_000, 250_000, n, dtype=np.int64), mask=rng.random(n) < 0.01)   # negative keys: sign-flip encoding
    vals = pa.array(rng.integers(-100, 101, n, dtype=np.int64), mask=rng.random(n) < 0.1)
    check_path(ctx, keys, vals, 500_000, "dense", offset=offset)
    check_path(ctx, keys, vals, 0, "dense", offset=offset)


def test_dense_group_by_types_null_groups_and_batches(ctx):
    n = 4_400_000
    rng = np.random.default_rng(SEED + 37)
    # a group whose every value is null must exist with sum = null, count = 0 (the `exists` bitmap)
    kk = rng.integers(0, 300_000, n, dtype=np.int64)
    vv = rng.integers(-5, 5, n, dtype=np.int64)
    check_path(ctx, pa.array(kk), pa.array(vv, mask=(kk % 7 == 0) | (rng.random(n) < 0.05)), 300_000, "dense")
    # narrow native types: int32 keys, int16 / uint8 values (window = the type's range)
    k32 = pa.array(rng.integers(-70000, 70000, n, dtype=np.int32), mask=rng.random(n) < 0.02)
    v16 = pa.array(rng.integers(-30000, 30000, n, dtype=np.int16), mask=rng.random(n) < 0.1)
    check_path(ctx, k32, v16, 140_000, "dense")
    ku16 = pa.array(rng.integers(0, 60000, n, dtype=np.uint16))
    vu8 = pa.array(rng.integers(0, 255, n, dtype=np.uint8), mask=rng.random(n) < 0.5)
    check_path(ctx, ku16, vu8, 0, "dense")
    # unsigned 64-bit values around 2^63: sums wrap exactly like the reference
    vu64 = pa.array(rng.integers(2**63, 2**63 + 1000, n, dtype=np.uint64), mask=rng.random(n) < 0.1)
    check_path(ctx, ku16, vu64, 60_000, "dense")
    # several consume() calls into one table
    k2 = pa.array(rng.integers(0, 900_000, 3 * n, dtype=np.int64))
    v2 = pa.array(rng.integers(-100, 100, 3 * n, dtype=np.int64), mask=rng.random(3 * n) < 0.1)
    check_path(ctx, k2, v2, 0, "dense", batches=3)


def test_dense_windows_are_verified_not_trusted(ctx):
    """both windows come from a 64Ki-row SAMPLE: a key or a value outside them (at an unsampled row) must send the batch
    to the partitioned path instead of corrupting a neighbour's state"""
    n = 4_500_000
    step = n // 65536
    rng = np.random.default_rng(SEED + 41)
    k = rng.integers(0, 400_000, n, dtype=np.int64)
    v = rng.integers(-100, 101, n, dtype=np.int64)
    m = rng.random(n) < 0.1
    assert 2_000_001 % step != 0 and 2_000_003 % step != 0
    k2 = k.copy()
    k2[2_000_001] = 900_000_000              # key far outside the sampled range
    check_path(ctx, pa.array(k2), pa.array(v, mask=m), 0, "compact")
    v2 = v.copy()
    v2[2_000_003] = 2**40                    # value far outside the sampled window -> dense and compact both refuse
    m2 = m.copy()
    m2[2_000_003] = False
    check_path(ctx, pa.array(k), pa.array(v2, mask=m2), 0, "general")
    k3 = k.copy()
    k3[2_000_001] = -5                       # just below the sampled minimum but inside the slack: still dense
    check_path(ctx, pa.array(k3), pa.array(v, mask=m), 0, "dense")


def test_dense_state_coexists_with_the_hash_table(ctx):
    """consume() calls that take different paths into one object: dense, dense with another window (the first state is
    flushed into the table), compact, general (full-range keys), and a merge of partial states -- finalize must join all"""
    rng = np.random.default_rng(SEED + 43)
    n = 4_300_000
    batches = [
        (rng.integers(0, 200_000, n, dtype=np.int64), "dense"),
        (rng.integers(100_000, 300_000, n, dtype=np.int64), "dense"),            # sample inside [0, 200k + slack)? no: new window
        (rng.integers(5_000_000, 5_400_000, n, dtype=np.int64), "dense"),        # disjoint window
        (rng.integers(0, 600_000, 2_500_000, dtype=np.int64), "compact"),        # < 2^22 rows: partitioned
        (np.concatenate([rng.integers(0, 600_000, 2_400_000, dtype=np.int64), [np.iinfo(np.int64).min, -1, np.iinfo(np.int64).max]]), "general"),
    ]
    g = bc.GroupBySumCount(pa.int64(), pa.int64(), ctx=ctx)
    all_k, all_v = [], []
    for kk, _ in batches:
        keys = pa.array(kk, mask=rng.random(len(kk)) < 0.01)
        vals = pa.array(rng.integers(-100, 101, len(kk), dtype=np.int64), mask=rng.random(len(kk)) < 0.1)
        g.consume(DeviceArray.from_arrow(keys, ctx), DeviceArray.from_arrow(vals, ctx))
        all_k.append(keys)
        all_v.append(vals)
    paths = g.path_counts()
    assert paths == {"dense": 3, "compact": 1, "general": 1, "atomic": 0}, paths
    # plus partial states of a sixth shard, merged the way the owner GPU does after the exchange
    k6 = pa.array(rng.integers(0, 700_000, 2_200_000, dtype=np.int64))
    v6 = pa.array(rng.integers(-100, 101, 2_200_000, dtype=np.int64), mask=rng.random(2_200_000) < 0.1)
    h = bc.GroupBySumCount(pa.int64(), pa.int64(), ctx=ctx)
    h.consume(DeviceArray.from_arrow(k6, ctx), DeviceArray.from_arrow(v6, ctx))
    g.merge(*h.finalize())
    all_k.append(k6)
    all_v.append(v6)
    k, s, c = [x.to_arrow() for x in g.finalize()]
    got = pa.table({"k": k, "v_sum": s, "v_count": c}).sort_by("k")
    want = reference(pa.concat_arrays(all_k), pa.concat_arrays(all_v))
    assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
    assert got["v_count"].combine_chunks().equals(want["v_count"].combine_chunks())
    assert got["v_sum"].combine_chunks().equals(want["v_sum"].combine_chunks())


# ---- hash_sum HashAggregateKernel consume through the dense path (group ids as keys) ----------------------------
def _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=None, **opts):
    """two consume calls, the second from an odd row offset, each of at least 2^22 rows when the input has 2^23 + 8.
    want_dense: whether each consume must take dense_sum_count_by_id, checked by the kernels it launched against the
    restated list (tests/packed_regimes.py)"""
    from . import packed_regimes as P
    agg = bc.HashAggregator("hash_sum", vals.type, ctx=ctx, **opts)
    agg.resize(groups)
    n = len(ids)
    dids, dv = DeviceArray.from_arrow(ids, ctx), DeviceArray.from_arrow(vals, ctx)
    half = n // 2 + 3
    idn = ids.to_numpy()
    vn = vals.fill_null(0).to_numpy()
    valid = np.asarray(vals.is_valid())
    lib = _cabi.lib()
    for lo, hi in ((0, half), (half, n)):
        before = lib.b2_launch_count()
        agg.consume(dv.slice(lo, hi - lo), dids.slice(lo, hi - lo))
        launched = lib.b2_launch_count() - before
        if want_dense is not None:
            plan = P.byid_plan(idn[lo:hi], groups, vn[lo:hi], valid[lo:hi], skip_nulls=opts.get("skip_nulls", True),
                               settings=P.Settings.from_env())
            assert (plan.dense is not None) == want_dense, plan.why
            assert launched == plan.launches(vals.type.bit_width // 8, hi - lo, groups), plan.why
    return agg.finalize().to_arrow()


def _want_sum(ids, vals, groups, skip_nulls=True):
    idn = ids.to_numpy()
    valid = np.asarray(vals.is_valid())
    v = vals.fill_null(0).to_numpy().astype(np.int64 if pa.types.is_signed_integer(vals.type) else np.uint64)
    sums = np.zeros(groups, dtype=v.dtype)
    np.add.at(sums, idn[valid], v[valid])
    counts = np.bincount(idn[valid], minlength=groups)
    ok = counts >= 1
    if not skip_nulls:
        ok &= np.bincount(idn[~valid], minlength=groups) == 0
    return pa.array(sums, mask=~ok)


def _by_id_input(vt, n, groups, seed):
    rng = np.random.default_rng(seed)
    ids = pa.array(rng.integers(0, groups - 7, n, dtype=np.uint32), pa.uint32())   # the last 7 groups stay empty -> null sums
    info = np.iinfo(vt.to_pandas_dtype())
    lo, hi = max(int(info.min), -1000), min(int(info.max), 1000)
    return ids, pa.array(rng.integers(lo, hi, n).astype(vt.to_pandas_dtype()), vt, mask=rng.random(n) < 0.1)


@pytest.mark.parametrize("vt", [pa.int64(), pa.uint16(), pa.uint64(), pa.int8(), pa.int16()], ids=str)
def test_hash_sum_consume_takes_the_dense_path(ctx, vt, monkeypatch):
    n, groups = (1 << 23) + 8, 300_000
    ids, vals = _by_id_input(vt, n, groups, SEED + 11)
    want = _want_sum(ids, vals, groups)
    assert _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=True).equals(want)
    monkeypatch.setenv("B2_GROUPBY_DENSE", "0")
    assert _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=False).equals(want)


def test_hash_sum_consume_int32_declines_the_dense_path(ctx):
    """32-bit values leave a sub-batch 2^15 rows (m = (63 - 32) / 2), too few for the packed state: the atomic kernel"""
    n, groups = (1 << 23) + 8, 300_000
    ids, vals = _by_id_input(pa.int32(), n, groups, SEED + 11)
    assert _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=False).equals(_want_sum(ids, vals, groups))


def test_hash_sum_dense_path_window_violation_and_skip_nulls_false(ctx):
    n, groups = (1 << 23) + 8, 200_000
    rng = np.random.default_rng(SEED + 12)
    ids = pa.array(rng.integers(0, groups, n, dtype=np.uint32), pa.uint32())
    v = rng.integers(-50, 50, n)
    # outside any sampled window, at rows the sample skips: each consume runs the dense path, which declines, and the
    # atomic kernel redoes the batch
    v[[17, n // 3, n - 5]] = [2**61, -(2**62), 2**62 + 12345]
    mask = rng.random(n) < 0.05
    mask[[17, n // 3, n - 5]] = False
    vals = pa.array(v, pa.int64(), mask=mask)
    assert _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=False).equals(_want_sum(ids, vals, groups))
    # skip_nulls = false needs the per-group has-null flags: stays on the atomic kernel, same contract as before
    got = _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=False, skip_nulls=False)
    assert got.equals(_want_sum(ids, vals, groups, skip_nulls=False))
    # without the outliers both consumes take the dense path
    v[[17, n // 3, n - 5]] = 0
    vals = pa.array(v, pa.int64(), mask=rng.random(n) < 0.05)
    assert _hash_sum_by_ids(ctx, ids, vals, groups, want_dense=True).equals(_want_sum(ids, vals, groups))


def test_grouper_aggregators_in_l2_bands(ctx):
    """hash_count / hash_min / hash_max / hash_mean through the Grouper path with more than 2^24 rows and 4M groups: the
    aggregators' state (32 to 64 MB) is consumed in several L2-sized bands of group ids (hash_aggregate.cu launch_consume)"""
    import pyarrow.acero  # noqa: F401
    n, groups = (1 << 24) + 4099, 4_000_000
    rng = np.random.default_rng(SEED + 24)
    keys = pa.array(rng.integers(0, groups, n, dtype=np.int64))
    vals = pa.array(rng.integers(-1000, 1000, n, dtype=np.int32), mask=rng.random(n) < 0.1)
    dk, dv = DeviceArray.from_arrow(keys, ctx), DeviceArray.from_arrow(vals, ctx)
    fns = ("hash_count", "hash_min", "hash_max", "hash_mean")
    (k,), outs = bc.group_by([dk], [(fn, dv, None) for fn in fns], fused=False)
    got = pa.table({"k": k.to_arrow(), **{fn: o.to_arrow() for fn, o in zip(fns, outs)}}).sort_by("k")
    want = pa.table({"k": keys, "v": vals}).group_by("k", use_threads=False).aggregate(
        [("v", "count"), ("v", "min"), ("v", "max"), ("v", "mean")]).sort_by("k")
    assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
    for fn, col in (("hash_count", "v_count"), ("hash_min", "v_min"), ("hash_max", "v_max")):
        assert got[fn].combine_chunks().equals(want[col].combine_chunks()), fn
    gm, wm = got["hash_mean"].combine_chunks(), want["v_mean"].combine_chunks()
    assert gm.is_valid().equals(wm.is_valid())
    np.testing.assert_allclose(gm.fill_null(0).to_numpy(), wm.fill_null(0).to_numpy(), rtol=1e-12)
