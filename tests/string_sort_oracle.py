"""The reference's sort over base-binary values, restated for the tests (the numeric cases are oracle/arrow_oracle.py's):
ArrayCompareSorter (kernels/vector_array_sort.cc:144-178) is std::stable_sort of the valid rows with `lhs < rhs` on the
raw bytes -- unsigned, a proper prefix first -- and `rhs < lhs` for Descending, so equal values keep index order either
way; nulls are stably partitioned to the end or the start.  sort_indices_multi and select_k_unstable follow the oracle's
own restatements (least significant key first; the stable sort's prefix), with string keys allowed."""
import numpy as np
import pyarrow as pa

from oracle import arrow_oracle as ora


def is_binary(t) -> bool:
    return pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t) or pa.types.is_large_binary(t)


def sort_indices(arr: pa.Array, order: str = "ascending", null_placement: str = "at_end") -> pa.Array:
    if not is_binary(arr.type):
        return ora.sort_indices(arr, order, null_placement)
    offs, data = ora.strings(arr)  # the oracle's own offsets / bytes helper
    valid = ora.validity(arr)
    vals = [data[offs[i]:offs[i + 1]].tobytes() for i in range(len(arr))]
    rows = [i for i in range(len(arr)) if valid[i]]
    rows.sort(key=lambda i: vals[i], reverse=order == "descending")  # Python's sort stays stable when reversed
    nulls = [i for i in range(len(arr)) if not valid[i]]
    out = rows + nulls if null_placement == "at_end" else nulls + rows
    return ora.make_array(pa.uint64(), np.array(out, dtype=np.uint64))


def select_k_unstable(arr: pa.Array, k: int, order: str = "ascending", null_placement: str = "at_end") -> pa.Array:
    if k < 0:
        raise pa.ArrowInvalid(f"select_k_unstable requires a nonnegative `k`, got {k}")
    return sort_indices(arr, order, null_placement).slice(0, min(k, len(arr)))


def sort_indices_multi(columns, sort_keys, null_placement: str = "at_end") -> pa.Array:
    n = len(next(iter(columns.values())))
    perm = np.arange(n, dtype=np.uint64)
    for name, order in reversed(list(sort_keys)):
        col = columns[name].take(pa.array(perm))
        perm = perm[ora.values(sort_indices(col, order, null_placement)).astype(np.int64)]
    return pa.array(perm, pa.uint64())
