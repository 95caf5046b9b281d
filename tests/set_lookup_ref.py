"""Exact host restatement of the reference's set lookup (cpp/src/arrow/compute/kernels/scalar_set_lookup.cc).

  state    SetLookupState::Init / AddArrayValueSet (:44-129): every distinct value -> the position of its first
           occurrence in the value set, positions continuing across chunks; null_index = the first null's position
           unless the behaviour is SKIP (then, or without a null, -1).  Numbers are keyed by their bit pattern at their
           width (UnsignedIntType<sizeof>), so -0.0 != +0.0 and NaNs match by payload; strings by bytes.
  is_in    IsInVisitor::ProcessIsIn (:435-475)
  index_in IndexInVisitor::ProcessIndexIn (:306-340); data under null slots is 0.

set_lookup() returns (data, valid) as numpy arrays -- bool data for is_in, int32 for index_in -- so a caller can check
the slots under nulls too; to_arrow() turns them into the pyarrow result.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

BEHAVIORS = ("match", "skip", "emit_null", "inconclusive")
_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _concat(arr) -> pa.Array:
    if isinstance(arr, pa.ChunkedArray):
        return pa.concat_arrays(arr.chunks) if arr.num_chunks else pa.array([], arr.type)
    return arr


def _valid(arr: pa.Array) -> np.ndarray:
    return np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)


def _fixed_bits(arr: pa.Array):
    """the values' bit patterns as unsigned integers of their width (slots under nulls included)"""
    w = arr.type.bit_width // 8
    buf = arr.buffers()[1]
    return np.frombuffer(buf, dtype=_UINT[w], count=arr.offset + len(arr))[arr.offset:]


def _is_fixed(t: pa.DataType) -> bool:
    return pa.types.is_integer(t) or pa.types.is_floating(t)


def state(value_set, behavior: str):
    """(keys, first positions, null_index): keys sorted (fixed width) or a dict key -> first position (others)"""
    vs = _concat(value_set)
    valid = _valid(vs)
    nulls = np.nonzero(~valid)[0]
    null_index = int(nulls[0]) if len(nulls) and behavior != "skip" else -1
    rows = np.nonzero(valid)[0]
    if _is_fixed(vs.type):
        keys, first = np.unique(_fixed_bits(vs)[rows], return_index=True)  # return_index: the first occurrence
        return keys, rows[first].astype(np.int64), null_index
    memo = {}
    for i, v in zip(rows.tolist(), vs.filter(pa.array(valid)).to_pylist()):
        memo.setdefault(v, i)
    return memo, None, null_index


def _positions(values: pa.Array, st) -> np.ndarray:
    """first position of every valid value in the value set, -1 where absent (and for null rows)"""
    keys, first, _ = st
    valid = _valid(values)
    if first is not None:
        bits = _fixed_bits(values)
        if len(keys) == 0:
            return np.full(len(values), -1, np.int64)
        j = np.minimum(np.searchsorted(keys, bits), len(keys) - 1)
        return np.where(valid & (keys[j] == bits), first[j], -1)
    return np.array([keys.get(v, -1) if ok else -1 for v, ok in zip(values.to_pylist(), valid)], dtype=np.int64)


def set_lookup(values: pa.Array, value_set, behavior: str, function: str):
    """(data, valid) of is_in / index_in for values and a value set of the same type"""
    assert behavior in BEHAVIORS, behavior
    st = state(value_set, behavior)
    null_index = st[2]
    has_null = null_index != -1
    valid_in = _valid(values)
    pos = _positions(values, st)
    found = pos >= 0
    if function == "index_in":
        null_match = behavior == "match" and has_null
        data = np.where(valid_in, np.where(found, pos, 0), null_index if null_match else 0).astype(np.int32)
        valid = np.where(valid_in, found, null_match)
        return data, valid
    assert function == "is_in", function
    miss_null = behavior == "inconclusive" and has_null
    null_true = behavior == "match" and has_null
    null_false = behavior == "skip" or (behavior == "match" and not has_null)
    data = np.where(valid_in, found, null_true)
    valid = np.where(valid_in, found | (not miss_null), null_true or null_false)
    return data.astype(bool), valid.astype(bool)


def to_arrow(data: np.ndarray, valid: np.ndarray, function: str) -> pa.Array:
    t = pa.int32() if function == "index_in" else pa.bool_()
    return pa.array(data, t, mask=~valid)


def expected(values: pa.Array, value_set, behavior: str, function: str) -> pa.Array:
    return to_arrow(*set_lookup(values, value_set, behavior, function), function)
