"""CPU checks of tests/groupings_ref.py, the reference every GPU groupings / hash_list / hash_distinct test compares
against: the MakeGroupings known answers of compute/row/grouper_test.cc:1274-1307, and pyarrow's own hash_list /
hash_distinct through group_by(use_threads=False) -- lists in exact order, distinct lists sorted inside each list (the
reference does not fix that order, hash_aggregate_test.cc:2487)."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import groupings_ref as gr

SEED = 0x6A0F


@pytest.mark.parametrize("ids, expected", [
    ([], [[]]),
    ([0, 0, 0], [[0, 1, 2]]),
    ([0, 0, 0, 1, 1, 2], [[0, 1, 2], [3, 4], [5], []]),
    ([2, 1, 2, 1, 1, 2], [[], [1, 3, 4], [0, 2, 5], [], []]),
    ([2, 2, 5, 5, 2, 3], [[], [], [0, 1, 4], [5], [], [2, 3], [], []]),
])
def test_make_groupings_known_answers(ids, expected):
    got = gr.make_groupings(pa.array(ids, pa.uint32()), len(expected))
    assert got.equals(pa.array(expected, pa.list_(pa.int32())))
    grouped = gr.apply_groupings(got, pa.array(ids, pa.uint32()))
    for g, sub in enumerate(grouped.to_pylist()):
        assert all(x == g for x in sub)


def test_make_groupings_refuses_null_ids():
    with pytest.raises(pa.ArrowInvalid, match="MakeGroupings with null ids"):
        gr.make_groupings(pa.array([0, None, 1], pa.uint32()), 5)


def test_make_groupings_refuses_ids_out_of_range():
    with pytest.raises(pa.ArrowIndexError):
        gr.make_groupings(pa.array([0, 5], pa.uint32()), 5)


def test_groups_never_consumed_are_empty():
    got = gr.hash_list(pa.array([1.5, None]), pa.array([1, 1], pa.uint32()), 4)
    assert got.to_pylist() == [[], [1.5, None], [], []]
    assert gr.hash_distinct(pa.array([1, 1, None]), pa.array([2, 2, 2], pa.uint32()), 3, "all").to_pylist() == [[], [], [1, None]]


def values_of(t, n, rng):
    """n values of type t with ~15% nulls, few distinct values (so hash_distinct has work), specials for floats"""
    mask = rng.random(n) < 0.15
    if pa.types.is_boolean(t):
        return pa.array(rng.random(n) < 0.5, mask=mask)
    if pa.types.is_floating(t):
        pool = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.5, -2.25, 3.0])
        return pa.array(pool[rng.integers(0, len(pool), n)].astype(t.to_pandas_dtype()), t, mask=mask)
    if pa.types.is_integer(t):
        info = np.iinfo(t.to_pandas_dtype())
        pool = np.array([info.min, info.max, 0, 1, 7], dtype=t.to_pandas_dtype())
        return pa.array(pool[rng.integers(0, len(pool), n)], t, mask=mask)
    if pa.types.is_date32(t) or pa.types.is_timestamp(t):
        raw = pa.array(rng.integers(-5, 5, n), pa.int64() if pa.types.is_timestamp(t) else pa.int32(), mask=mask)
        return raw.cast(t)
    if pa.types.is_fixed_size_binary(t):
        words = [bytes([i % 3]) * t.byte_width for i in range(6)]
        return pa.array([None if m else words[k] for m, k in zip(mask, rng.integers(0, 6, n))], t)
    words = ["", "a", "bb", "é", "a\x00", "zzzzzzzzzzzz"]
    items = [None if m else words[k] for m, k in zip(mask, rng.integers(0, len(words), n))]
    if pa.types.is_binary(t) or pa.types.is_large_binary(t):
        items = [None if x is None else x.encode() for x in items]
    return pa.array(items, t)


LIST_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64(),
              pa.float32(), pa.float64(), pa.date32(), pa.timestamp("us"), pa.bool_(), pa.string(), pa.binary(),
              pa.large_string(), pa.large_binary(), pa.binary(4), pa.binary(16)]
DISTINCT_TYPES = [t for t in LIST_TYPES if not pa.types.is_boolean(t) and not pa.types.is_fixed_size_binary(t)]


def dense_ids(keys: pa.Array) -> pa.Array:
    """first-occurrence group ids, as the Grouper assigns them"""
    return pc.dictionary_encode(keys).indices.cast(pa.uint32())


def pyarrow_group_by(keys, values, agg, options=None):
    tbl = pa.table({"k": keys, "v": values})
    out = tbl.group_by("k", use_threads=False).aggregate([("v", agg, options)] if options else [("v", agg)])
    return out.column(f"v_{agg}").combine_chunks()


def sort_inside(lists: pa.Array):
    """each list as its sorted element reprs: NaN equals NaN, -0.0 differs from 0.0"""
    return [sorted(map(repr, sub)) for sub in lists.to_pylist()]


def inputs(t, n, offset, seed):
    rng = np.random.default_rng(seed)
    keys = pa.array(rng.integers(0, 5, n + offset + 3), pa.int64()).slice(offset, n)
    values = values_of(t, n + offset + 3, rng).slice(offset, n)
    return keys, values


@pytest.mark.parametrize("t", LIST_TYPES, ids=str)
@pytest.mark.parametrize("n, offset", [(0, 0), (200, 0), (200, 3), (77, 13)])
def test_hash_list_matches_pyarrow(t, n, offset):
    keys, values = inputs(t, n, offset, SEED + n + offset)
    ids = dense_ids(keys)
    want = pyarrow_group_by(keys, values, "list")
    got = gr.hash_list(values, ids, len(want))
    gr.assert_same_lists(got, want)


@pytest.mark.parametrize("t", DISTINCT_TYPES, ids=str)
@pytest.mark.parametrize("mode", ["only_valid", "only_null", "all"])
@pytest.mark.parametrize("n, offset", [(0, 0), (200, 0), (77, 13)])
def test_hash_distinct_matches_pyarrow(t, mode, n, offset):
    keys, values = inputs(t, n, offset, SEED + 7 * n + offset)
    ids = dense_ids(keys)
    want = pyarrow_group_by(keys, values, "distinct", pc.CountOptions(mode))
    got = gr.hash_distinct(values, ids, len(want), mode)
    assert sort_inside(got) == sort_inside(want)
