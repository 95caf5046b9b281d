"""Group-major order (Grouper.make_groupings / apply_groupings) and the list-valued hash aggregates hash_list /
hash_distinct on the device, against tests/groupings_ref.py (exact order) and pyarrow's group_by(use_threads=False)
(hash_list exact, hash_distinct sorted inside each list)."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import groupings_ref as gr
from tests.test_groupings_oracle import DISTINCT_TYPES, LIST_TYPES, dense_ids, pyarrow_group_by, sort_inside, values_of

pytestmark = pytest.mark.gpu
SEED = 0x6A0F
TILE = 4096  # rows per onesweep tile


def dev(a, ctx):
    return DeviceArray.from_arrow(a, ctx)


@pytest.mark.parametrize("groups", [1, 256, 257, 65536, 65537, (1 << 24) + 1])
@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_make_groupings_matches_reference(ctx, groups, n):
    rng = np.random.default_rng(SEED + groups + n)
    ids = rng.integers(0, groups, n).astype(np.uint32)
    if n > 1:
        ids[0], ids[-1] = 0, groups - 1  # every digit of the largest id varies
    want = gr.make_groupings(pa.array(ids, pa.uint32()), groups)
    got = bc.Grouper.make_groupings(dev(pa.array(ids, pa.uint32()), ctx), groups).to_arrow()
    assert got.equals(want)


@pytest.mark.parametrize("offset", [3, 13])
def test_make_groupings_sliced_ids(ctx, offset):
    rng = np.random.default_rng(SEED + offset)
    full = pa.array(rng.integers(0, 300, 3 * TILE).astype(np.uint32), pa.uint32())
    ids = full.slice(offset, 2 * TILE + 5)
    got = bc.Grouper.make_groupings(dev(full, ctx).slice(offset, 2 * TILE + 5), 301).to_arrow()
    assert got.equals(gr.make_groupings(ids, 301))


def test_make_groupings_edges(ctx):
    empty = dev(pa.array([], pa.uint32()), ctx)
    assert bc.Grouper.make_groupings(empty, 0).to_arrow().to_pylist() == []
    assert bc.Grouper.make_groupings(empty, 3).to_arrow().to_pylist() == [[], [], []]
    same = dev(pa.array([7] * 5000, pa.uint32()), ctx)  # one distinct id: no radix pass runs
    assert bc.Grouper.make_groupings(same, 9).to_arrow().equals(gr.make_groupings(pa.array([7] * 5000, pa.uint32()), 9))
    for ids, expected in [([0, 0, 0, 1, 1, 2], [[0, 1, 2], [3, 4], [5], []]),
                          ([2, 2, 5, 5, 2, 3], [[], [], [0, 1, 4], [5], [], [2, 3], [], []])]:
        g = bc.Grouper.make_groupings(dev(pa.array(ids, pa.uint32()), ctx), len(expected))
        assert g.to_arrow().to_pylist() == expected
        applied = bc.Grouper.apply_groupings(g, dev(pa.array(ids, pa.uint32()), ctx)).to_arrow()
        assert applied.to_pylist() == [[i] * len(sub) for i, sub in enumerate(expected)]


def test_make_groupings_errors(ctx):
    with pytest.raises(pa.ArrowInvalid, match="MakeGroupings with null ids"):
        bc.Grouper.make_groupings(dev(pa.array([0, None, 1], pa.uint32()), ctx), 5)
    with pytest.raises(pa.ArrowIndexError):
        bc.Grouper.make_groupings(dev(pa.array([0, 5, 1], pa.uint32()), ctx), 5)
    with pytest.raises(pa.ArrowIndexError):
        bc.Grouper.make_groupings(dev(pa.array(np.arange(70000, dtype=np.uint32)), ctx), 65536)


def test_make_groupings_capacity(ctx):
    import torch
    torch.cuda.synchronize()
    n = (1 << 31)  # INT32_MAX + 1 real ids
    buf = torch.zeros(n, dtype=torch.int32, device="cuda")
    ids = DeviceArray.from_pointers(ctx, pa.uint32(), n, buf.data_ptr(), keepalive=buf)
    with pytest.raises(pa.ArrowCapacityError):
        bc.Grouper.make_groupings(ids, 1)
    del ids, buf
    torch.cuda.empty_cache()


def test_make_groupings_beyond_2_30_rows(ctx):
    """2^30 + 5 ids over 10M groups (three radix passes, 64-bit look-back cells), checked on the device with torch"""
    import torch

    from tests.test_gpu_fullsize import as_tensor
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()
    n, groups = (1 << 30) + 5, 10_000_000
    gen = torch.Generator(device="cuda").manual_seed(SEED)
    ids_t = torch.randint(0, groups, (n,), dtype=torch.int32, device="cuda", generator=gen)
    ids = DeviceArray.from_pointers(ctx, pa.uint32(), n, ids_t.data_ptr(), keepalive=ids_t)
    torch.cuda.synchronize()
    g = bc.Grouper.make_groupings(ids, groups)
    ctx.sync()
    rows = as_tensor(torch, g.children[0], torch.int32)
    offsets = as_tensor(torch, g, torch.int32, groups + 1)
    want = torch.zeros(groups + 1, dtype=torch.int64, device="cuda")
    want[1:] = torch.cumsum(torch.bincount(ids_t, minlength=groups), 0)
    assert torch.equal(offsets.to(torch.int64), want)
    seen = torch.zeros(n, dtype=torch.bool, device="cuda")
    chunk = 1 << 28
    prev_id = prev_row = None
    for lo in range(0, n, chunk):
        r = rows[lo:lo + chunk].to(torch.int64)
        seen[r] = True
        gid = ids_t[r]
        if prev_id is not None:
            gid = torch.cat([prev_id, gid])
            r = torch.cat([prev_row, r])
        assert bool((gid[1:] >= gid[:-1]).all()), "ids decrease along the output"
        same = gid[1:] == gid[:-1]
        assert bool((r[1:][same] > r[:-1][same]).all()), "rows do not increase inside a group"
        prev_id, prev_row = gid[-1:], r[-1:]
        del r, gid, same
    assert bool(seen.all()), "a row is missing"
    del g, rows, offsets, seen, ids, ids_t
    torch.cuda.empty_cache()


# ---- hash_list / hash_distinct ---------------------------------------------------------------------------------------
def keyed(t, n, seed, n_keys=7):
    rng = np.random.default_rng(seed)
    keys = pa.array(rng.integers(0, n_keys, n + 11), pa.int64()).slice(5, n)
    values = values_of(t, n + 11, rng).slice(5, n)
    return keys, values


def run_agg(ctx, fn, t, batches, groups, mode="only_valid", merge=None):
    """batches: [(values, ids)] consumed in order; merge: (batches, groups, mapping) of a second state merged after"""
    opts = {"mode": mode} if fn == "hash_distinct" else {}
    agg = bc.HashAggregator(fn, t, ctx=ctx, **opts)
    agg.resize(groups)
    for v, i in batches:
        agg.consume(dev(v, ctx), dev(i, ctx))
    if merge is not None:
        other_batches, other_groups, mapping = merge
        other = bc.HashAggregator(fn, t, ctx=ctx, **opts)
        other.resize(other_groups)
        for v, i in other_batches:
            other.consume(dev(v, ctx), dev(i, ctx))
        agg.merge(other, dev(pa.array(mapping, pa.uint32()), ctx))
    out = agg.finalize()
    assert pa.types.is_list(out.type) and out.type.value_type == t
    return out.to_arrow()


def expected(fn, values, ids, groups, mode):
    return gr.hash_list(values, ids, groups) if fn == "hash_list" else gr.hash_distinct(values, ids, groups, mode)


CASES = [("hash_list", t, "only_valid") for t in LIST_TYPES] + \
        [("hash_distinct", t, m) for t in DISTINCT_TYPES for m in ("only_valid", "only_null", "all")]


@pytest.mark.parametrize("fn, t, mode", CASES, ids=lambda x: str(x))
def test_one_consume(ctx, fn, t, mode):
    keys, values = keyed(t, 3000, SEED + len(str(t)))
    ids = dense_ids(keys)
    groups = len(pc.unique(keys)) + 2  # two groups never consumed
    got = run_agg(ctx, fn, t, [(values, ids)], groups, mode)
    gr.assert_same_lists(got, expected(fn, values, ids, groups, mode))
    agg = "list" if fn == "hash_list" else "distinct"
    want = pyarrow_group_by(keys, values, agg, pc.CountOptions(mode) if fn == "hash_distinct" else None)
    head = got.slice(0, groups - 2)
    if fn == "hash_list":
        gr.assert_same_lists(head, want)
    else:
        assert sort_inside(head) == sort_inside(want)


@pytest.mark.parametrize("fn, t, mode", CASES, ids=lambda x: str(x))
def test_several_consumes(ctx, fn, t, mode):
    keys, values = keyed(t, 5000, SEED + 3 * len(str(t)))
    ids = dense_ids(keys)
    groups = len(pc.unique(keys))
    cuts = [0, 13, 1300, 1301, 5000]  # batches at bit offsets that are not multiples of 8
    batches = [(values.slice(a, b - a), ids.slice(a, b - a)) for a, b in zip(cuts, cuts[1:])]
    got = run_agg(ctx, fn, t, batches, groups, mode)
    gr.assert_same_lists(got, expected(fn, values, ids, groups, mode))


@pytest.mark.parametrize("fn, t, mode", CASES, ids=lambda x: str(x))
def test_merge_reversed_mapping(ctx, fn, t, mode):
    keys, values = keyed(t, 4000, SEED + 5 * len(str(t)))
    groups = 7
    ids = pa.array(np.asarray(keys), pa.uint32())
    a_v, a_i, b_v, b_i = values.slice(0, 1501), ids.slice(0, 1501), values.slice(1501), ids.slice(1501)
    mapping = np.arange(groups, dtype=np.uint32)[::-1].copy()
    got = run_agg(ctx, fn, t, [(a_v, a_i)], groups, mode, merge=([(b_v, b_i)], groups, mapping))
    # this state's rows, then the other state's with its ids mapped
    all_v = pa.concat_arrays([a_v, b_v])
    all_i = pa.array(np.concatenate([np.asarray(a_i), mapping[np.asarray(b_i)]]), pa.uint32())
    gr.assert_same_lists(got, expected(fn, all_v, all_i, groups, mode))


def test_group_by_path(ctx):
    rng = np.random.default_rng(SEED)
    keys = pa.array(rng.integers(0, 50, 20000), pa.int64())
    words = pa.array([None if x % 9 == 0 else f"w{x % 37}" for x in rng.integers(0, 1000, 20000)], pa.string())
    nums = pa.array(rng.normal(size=20000), mask=rng.random(20000) < 0.1)
    uniq, (lst, dst) = bc.group_by([dev(keys, ctx)], [("hash_list", dev(nums, ctx), None),
                                                      ("hash_distinct", dev(words, ctx), {"mode": "all"})])
    tbl = pa.table({"k": keys, "n": nums, "w": words}).group_by("k", use_threads=False).aggregate(
        [("n", "list"), ("w", "distinct", pc.CountOptions("all"))])
    assert uniq[0].to_arrow().equals(tbl["k"].combine_chunks())
    gr.assert_same_lists(lst.to_arrow(), tbl["n_list"].combine_chunks())
    assert sort_inside(dst.to_arrow()) == sort_inside(tbl["w_distinct"].combine_chunks())


def test_list_device_array_round_trip_and_refusals(ctx):
    arr = pa.array([[1, None], [], None, [4, 5, 6]], pa.list_(pa.int64()))
    d = dev(arr, ctx)
    assert d.to_arrow().equals(arr)
    assert d.slice(1, 3).to_arrow().equals(arr.slice(1, 3))
    idx = dev(pa.array([0, 1], pa.int32()), ctx)
    mask = dev(pa.array([True, False, True, True]), ctx)
    refused = (pa.ArrowNotImplementedError, pa.ArrowTypeError, pa.ArrowInvalid)
    for call in (lambda: bc.take(d, idx), lambda: bc.filter(d, mask), lambda: bc.array_sort_indices(d),
                 lambda: bc.unique(d), lambda: bc.Grouper([arr.type], ctx),
                 lambda: bc.HashAggregator("hash_sum", arr.type, ctx=ctx),
                 lambda: bc.HashAggregator("hash_list", arr.type, ctx=ctx)):
        with pytest.raises(refused):
            call()


def test_list_finalize_entry_points_are_separate(ctx):
    agg = bc.HashAggregator("hash_list", pa.int32(), ctx=ctx)
    agg.resize(1)
    with pytest.raises(pa.ArrowInvalid, match="b2_hashagg_finalize_list"):
        from arrow_b200 import _cabi as cabi
        import ctypes as C
        from arrow_b200.device import check
        out = cabi.B2Array()
        check(ctx.lib.b2_hashagg_finalize(agg.handle, C.byref(out), ctx.stream))


def test_hash_list_ids_out_of_range(ctx):
    agg = bc.HashAggregator("hash_list", pa.int32(), ctx=ctx)
    agg.resize(2)
    agg.consume(dev(pa.array([1, 2, 3], pa.int32()), ctx), dev(pa.array([0, 1, 2], pa.uint32()), ctx))
    with pytest.raises(pa.ArrowIndexError):
        agg.finalize()


@pytest.mark.parametrize("fn, t, mode", CASES, ids=lambda x: str(x))
def test_zero_rows(ctx, fn, t, mode):
    """resize alone, then a zero-row batch: num_groups empty lists of the value type"""
    empty_v, empty_i = values_of(t, 0, np.random.default_rng(0)), pa.array([], pa.uint32())
    for batches in ([], [(empty_v, empty_i)]):
        got = run_agg(ctx, fn, t, batches, 3, mode)
        assert got.to_pylist() == [[], [], []]


def test_make_groupings_sparse_ids(ctx):
    """a few ids spread over many groups: every gap between run boundaries is long (the binary-search offsets)"""
    groups = 50_000_000
    ids = np.array([groups - 1, 7, 7, 1_000_000, 30_000_000, 0, 1_000_001, groups - 1], np.uint32)
    got = bc.Grouper.make_groupings(dev(pa.array(ids, pa.uint32()), ctx), groups)
    offsets = np.frombuffer(got.buffers[1].to_numpy(4 * (groups + 1)), np.int32)
    want = np.zeros(groups + 1, np.int64)
    want[1:] = np.cumsum(np.bincount(ids, minlength=groups))
    assert np.array_equal(offsets, want)
    assert got.children[0].to_arrow().to_pylist() == np.argsort(ids, kind="stable").tolist()
