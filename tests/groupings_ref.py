"""numpy restatement of the reference's group-major order and the list-valued hash aggregates.

The reference (arrow/compute):
  * Grouper::MakeGroupings (row/grouper.h:141-167, row/grouper.cc:986-1025): list<int32> of length num_groups, entry g =
    the rows whose id is g in row order (a stable counting sort); null ids are Invalid;
  * Grouper::ApplyGroupings (grouper.h:169-194, grouper.cc:975-984): Take(values, groupings.values) under the groupings'
    offsets;
  * hash_list (kernels/hash_aggregate.cc:1858-2047): every (value, id) row, nulls kept, consume order then merge order;
    Finalize = MakeGroupings + ApplyGroupings;
  * hash_distinct (hash_aggregate.cc:1400-1539): a Grouper over (value, id) -- keys compare by their bytes, so NaN
    payloads and signed zeros stay apart -- and the pairs' first-occurrence order; CountOptions mode ONLY_VALID drops
    the null, ONLY_NULL keeps only it, ALL keeps every pair.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa


def make_groupings(ids, num_groups: int) -> pa.ListArray:
    ids = pa.array(ids, pa.uint32()) if not isinstance(ids, pa.Array) else ids
    if ids.null_count:
        raise pa.ArrowInvalid("MakeGroupings with null ids")
    a = ids.to_numpy(zero_copy_only=False).astype(np.int64)
    if len(a) and a.max() >= num_groups:
        raise pa.ArrowIndexError("MakeGroupings: a group id is >= num_groups")
    rows = np.argsort(a, kind="stable").astype(np.int32)
    offsets = np.zeros(num_groups + 1, np.int32)
    np.cumsum(np.bincount(a, minlength=num_groups), out=offsets[1:])
    return pa.ListArray.from_arrays(pa.array(offsets, pa.int32()), pa.array(rows, pa.int32()))


def apply_groupings(groupings: pa.ListArray, values: pa.Array) -> pa.ListArray:
    child = values.take(groupings.values)
    return pa.ListArray.from_arrays(groupings.offsets, child, type=pa.list_(values.type))


def hash_list(values: pa.Array, ids, num_groups: int) -> pa.ListArray:
    """values / ids: the rows in consume order (concatenate the batches, then the merged states' rows)"""
    return apply_groupings(make_groupings(ids, num_groups), values)


def _keys(values: pa.Array):
    """hashable key per row with the Grouper's equality: value bits for floats, None for null"""
    valid = np.asarray(values.is_valid())
    t = values.type
    if pa.types.is_floating(t):
        width = {16: np.uint16, 32: np.uint32, 64: np.uint64}[t.bit_width]
        bits = values.fill_null(0).to_numpy(zero_copy_only=False).view(width)
        return [int(b) if v else None for b, v in zip(bits, valid)]
    return [x if v else None for x, v in zip(values.to_pylist(), valid)]


def distinct_pairs(values: pa.Array, ids):
    """(first row of each distinct (value, id) pair) in first-occurrence order"""
    ids = np.asarray(pa.array(ids, pa.uint32()) if not isinstance(ids, pa.Array) else ids, dtype=np.int64)
    seen, firsts = set(), []
    for i, (k, g) in enumerate(zip(_keys(values), ids)):
        if (k, g) not in seen:
            seen.add((k, g))
            firsts.append(i)
    return np.asarray(firsts, np.int64)


def hash_distinct(values: pa.Array, ids, num_groups: int, mode: str = "only_valid") -> pa.ListArray:
    ids = np.asarray(pa.array(ids, pa.uint32()) if not isinstance(ids, pa.Array) else ids, dtype=np.int64)
    firsts = distinct_pairs(values, ids)
    pv = values.take(pa.array(firsts, pa.int64()))
    pg = ids[firsts]
    if mode != "all":
        keep = np.asarray(pv.is_valid()) if mode == "only_valid" else ~np.asarray(pv.is_valid())
        pv = pv.filter(pa.array(keep))
        pg = pg[keep]
    return hash_list(pv, pa.array(pg, pa.uint32()), num_groups)


def assert_same_lists(got: pa.Array, want: pa.Array) -> None:
    """equal list arrays, float children compared by their bits (NaN == NaN, -0.0 != 0.0)"""
    got, want = got.cast(want.type) if got.type != want.type else got, want
    assert len(got) == len(want) and got.null_count == want.null_count == 0
    assert np.array_equal(np.asarray(got.offsets) - got.offsets[0].as_py(), np.asarray(want.offsets) - want.offsets[0].as_py())
    gv, wv = got.flatten(), want.flatten()
    if pa.types.is_floating(want.type.value_type):
        assert np.array_equal(np.asarray(gv.is_valid()), np.asarray(wv.is_valid()))
        assert _keys(gv) == _keys(wv)
    else:
        assert gv.equals(wv), f"{gv.to_pylist()[:20]} != {wv.to_pylist()[:20]}"
