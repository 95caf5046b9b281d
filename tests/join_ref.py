"""Row-at-a-time reference for the hash join with null-equal keys and a residual filter (acero HashJoinNode with
JoinKeyCmp::IS and HashJoinNodeOptions::filter; JoinResidualFilter, acero/swiss_join_internal.h).

hash_join_indices(left_keys, right_keys, join_type, key_cmp, residual) gives the exact order and layout of
arrow_b200.compute.hash_join_indices: left rows in row order, the surviving matches of a left row in right-row order, the
null-extended row of an outer join in place of a left row's empty list, FULL OUTER's right rows with no surviving pair
last, in row order."""
import pyarrow as pa

from oracle.arrow_oracle import Grouper

JOIN_TYPES = ("inner", "left outer", "left semi", "left anti", "full outer")


def hash_join_indices(left_keys, right_keys, join_type: str = "inner", key_cmp=None, residual=None):
    """key_cmp: None (all "eq") or one "eq" / "is" per key column -- with "eq" a null key matches nothing, with "is" a
    null equals a null.  residual(l, r) -> True / False / None for the key-matching pair (left row l, right row r); a
    pair survives only on True.  Returns (left rows, right rows or None) as uint32 arrays, None standing for a null index;
    "left semi" / "left anti" return (left rows, None)."""
    if join_type not in JOIN_TYPES:
        raise ValueError(join_type)
    if isinstance(left_keys, pa.Array):
        left_keys, right_keys = [left_keys], [right_keys]
    cmp = list(key_cmp) if key_cmp is not None else ["eq"] * len(left_keys)
    eq_cols = [j for j, c in enumerate(cmp) if c == "eq"]
    lrows = list(Grouper([k.type for k in left_keys])._rows(left_keys))
    rrows = list(Grouper([k.type for k in right_keys])._rows(right_keys))

    def matchable(row):  # a null in an EQ column excludes the row
        return all(row[j] is not None for j in eq_cols)

    table = {}
    for j, row in enumerate(rrows):
        if matchable(row):
            table.setdefault(row, []).append(j)
    left, right = [], []
    hit_right = set()
    for i, row in enumerate(lrows):
        hits = table.get(row, []) if matchable(row) else []
        if residual is not None:
            hits = [j for j in hits if residual(i, j) is True]
        hit_right.update(hits)
        if join_type == "inner":
            left += [i] * len(hits)
            right += hits
        elif join_type in ("left outer", "full outer"):
            left += [i] * max(1, len(hits))
            right += hits if hits else [None]
        elif join_type == "left semi":
            left += [i] if hits else []
        else:
            left += [] if hits else [i]
    if join_type == "full outer":
        lonely = [j for j in range(len(rrows)) if j not in hit_right]
        left += [None] * len(lonely)
        right += lonely
    li = pa.array(left, pa.uint32())
    if join_type in ("left semi", "left anti"):
        return li, None
    return li, pa.array(right, pa.uint32())


def pairs_table(left: pa.Table, right: pa.Table, li: pa.Array, ri, left_cols, right_cols) -> pa.Table:
    """The join's output columns gathered through the index arrays (null index -> null row), as HashJoinNode emits them."""
    cols, names = [], []
    for n in left_cols:
        cols.append(left[n].combine_chunks().take(li))
        names.append(n)
    for n in right_cols:
        cols.append(right[n].combine_chunks().take(ri))
        names.append(n)
    return pa.table(cols, names=names)
