"""CPU checks of the join reference with a residual filter and null-equal keys (tests/join_ref.py): against pyarrow's own
hashjoin node with filter_expression for all eight join types, and against the reference's expected rows for
JoinKeyCmp::IS and the key / filter grid of its residual-filter test (tests/golden/kat_join_residual.json)."""
import json
import os
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.acero as acero
import pyarrow.compute as pc
import pytest

from tests import join_ref

HERE = os.path.dirname(os.path.abspath(__file__))
KAT = json.load(open(os.path.join(HERE, "golden", "kat_join_residual.json")))

ACERO_TYPES = ("inner", "left outer", "right outer", "full outer", "left semi", "right semi", "left anti", "right anti")
SWAPPED = {"right outer": "left outer", "right semi": "left semi", "right anti": "left anti"}


def rows_key(rows):
    return sorted(rows, key=repr)


def ref_pairs(lkeys, rkeys, join_type, key_cmp=None, residual=None):
    """(left row, right row) pairs of join_type (the eight acero types) from the reference; RIGHT_* through the swapped
    sides.  Semi / anti joins give (row, None) of the side they keep."""
    if join_type in SWAPPED:
        swapped = None if residual is None else (lambda r, l: residual(l, r))
        a, b = join_ref.hash_join_indices(rkeys, lkeys, SWAPPED[join_type], key_cmp, swapped)
        a = a.to_pylist()
        if b is None:
            return [(None, x) for x in a]
        return [(y, x) for x, y in zip(a, b.to_pylist())]
    a, b = join_ref.hash_join_indices(lkeys, rkeys, join_type, key_cmp, residual)
    a = a.to_pylist()
    return [(x, None) for x in a] if b is None else list(zip(a, b.to_pylist()))


def acero_pairs(left: pa.Table, right: pa.Table, lk, rk, join_type, filt):
    lt = left.append_column("_l", pa.array(np.arange(len(left), dtype=np.int64)))
    rt = right.append_column("_r", pa.array(np.arange(len(right), dtype=np.int64)))
    lout = [] if join_type in ("right semi", "right anti") else ["_l"]
    rout = [] if join_type in ("left semi", "left anti") else ["_r"]
    opts = acero.HashJoinNodeOptions(join_type, lk, rk, left_output=lout, right_output=rout, filter_expression=filt)
    decl = acero.Declaration("hashjoin", opts, inputs=[acero.Declaration("table_source", acero.TableSourceNodeOptions(lt)),
                                                       acero.Declaration("table_source", acero.TableSourceNodeOptions(rt))])
    t = decl.to_table(use_threads=False)
    ls = t["_l"].to_pylist() if lout else [None] * len(t)
    rs = t["_r"].to_pylist() if rout else [None] * len(t)
    return list(zip(ls, rs))


# ---- seeded many-to-many inputs with nulls on both sides ----
def make_sides(key_kind: str, seed: int, nl: int = 90, nr: int = 70):
    rng = np.random.default_rng(seed)

    def side(n, prefix):
        cols = {}
        if key_kind == "int64":
            cols[prefix + "k"] = pa.array(rng.integers(0, 9, n), pa.int64(), mask=rng.random(n) < 0.15)
        elif key_kind == "utf8":
            cols[prefix + "k"] = pa.array([f"key{v}" for v in rng.integers(0, 9, n)], pa.utf8(), mask=rng.random(n) < 0.15)
        else:
            cols[prefix + "k"] = pa.array(rng.integers(0, 3, n), pa.int64(), mask=rng.random(n) < 0.1)
            cols[prefix + "k2"] = pa.array([f"s{v}" for v in rng.integers(0, 3, n)], pa.utf8(), mask=rng.random(n) < 0.1)
        cols[prefix + "v"] = pa.array(rng.normal(size=n), pa.float64(), mask=rng.random(n) < 0.2)
        cols[prefix + "g"] = pa.array(rng.integers(0, 4, n), pa.int32())
        return pa.table(cols)

    left, right = side(nl, "l"), side(nr, "r")
    keys = ["k"] if key_kind != "two" else ["k", "k2"]
    return left, right, ["l" + k for k in keys], ["r" + k for k in keys]


def predicates(left: pa.Table, right: pa.Table, key_kind: str):
    """(name, acero expression, residual(l, r) -> True / False / None)"""
    lv, rv, lg = left["lv"].to_pylist(), right["rv"].to_pylist(), left["lg"].to_pylist()
    lk = left["lk"].to_pylist()

    def less(l, r):
        return None if lv[l] is None or rv[r] is None else lv[l] < rv[r]

    if key_kind == "utf8":
        key_expr, key_fn = pc.field("lk") > "key4", (lambda l, r: None if lk[l] is None else lk[l] > "key4")
    else:
        key_expr, key_fn = pc.field("lk") > 1, (lambda l, r: None if lk[l] is None else lk[l] > 1)
    return [
        ("payload_across_sides", pc.field("lv") < pc.field("rv"), less),
        ("key_referencing", key_expr, key_fn),
        ("literal_false", pc.scalar(False), lambda l, r: False),
        ("literal_true", pc.scalar(True), lambda l, r: True),
        ("fails_some_left_rows", pc.field("lg") != 0, lambda l, r: lg[l] != 0),
    ]


@pytest.mark.parametrize("key_kind", ["int64", "utf8", "two"])
@pytest.mark.parametrize("join_type", ACERO_TYPES)
def test_reference_matches_pyarrow_residual_filter(key_kind, join_type):
    left, right, lk, rk = make_sides(key_kind, seed=zlib.crc32(f"{key_kind}/{join_type}".encode()))
    for name, expr, fn in predicates(left, right, key_kind):
        want = acero_pairs(left, right, lk, rk, join_type, expr)
        got = ref_pairs([left[c].combine_chunks() for c in lk], [right[c].combine_chunks() for c in rk], join_type, residual=fn)
        assert rows_key(got) == rows_key(want), (name, join_type, key_kind)


def test_reference_orders_pairs_by_left_row_then_right_row():
    left, right, lk, rk = make_sides("int64", seed=7)
    lv, rv = left["lv"].to_pylist(), right["rv"].to_pylist()
    fn = lambda l, r: None if lv[l] is None or rv[r] is None else lv[l] < rv[r]  # noqa: E731
    li, ri = join_ref.hash_join_indices(left["lk"].combine_chunks(), right["rk"].combine_chunks(), "full outer", residual=fn)
    pairs = list(zip(li.to_pylist(), ri.to_pylist()))
    head = [p for p in pairs if p[0] is not None]
    tail = [p for p in pairs if p[0] is None]
    assert pairs == head + tail
    assert head == sorted(head, key=lambda p: (p[0], -1 if p[1] is None else p[1]))
    assert [r for _, r in tail] == sorted(r for _, r in tail)


# ---- the reference's expected rows ----
def _gather(rows, idx):
    return [None] * len(rows[0]) if idx is None else rows[idx]


def test_null_equal_full_outer_kat():
    case = KAT["is_full_outer"]
    lkey = pa.array(case["left"]["key"], pa.utf8())
    rkey = pa.array(case["right"]["key"], pa.utf8())
    li, ri = join_ref.hash_join_indices([lkey], [rkey], "full outer", key_cmp=case["key_cmp"])
    got = []
    for l, r in zip(li.to_pylist(), ri.to_pylist()):
        got.append((None if l is None else case["left"]["key"][l], None if l is None else case["left"]["payload"][l],
                    None if r is None else case["right"]["key"][r], None if r is None else case["right"]["payload"][r]))
    e = case["expected"]
    want = list(zip(e["l_key"], e["l_payload"], e["r_key"], e["r_payload"]))
    assert rows_key(got) == rows_key(want)
    # EQ: the null keys match nothing, so every null-key row is alone
    li, ri = join_ref.hash_join_indices([lkey], [rkey], "full outer", key_cmp=["eq"])
    assert sum(1 for l, r in zip(li.to_pylist(), ri.to_pylist()) if l is not None and r is not None) == 2


def test_null_equal_mixed_columns():
    """IS on one column, EQ on the other: a null in the IS column still matches, a null in the EQ column does not."""
    a = pa.array([None, None, 1, 1], pa.int64())
    b = pa.array([5, None, None, 5], pa.int64())
    li, ri = join_ref.hash_join_indices([a, b], [a, b], "inner", key_cmp=["is", "eq"])
    assert list(zip(li.to_pylist(), ri.to_pylist())) == [(0, 0), (3, 3)]
    li, ri = join_ref.hash_join_indices([a, b], [a, b], "inner", key_cmp=["is", "is"])
    assert list(zip(li.to_pylist(), ri.to_pylist())) == [(0, 0), (1, 1), (2, 2), (3, 3)]


GRID_FILTERS = {
    "true": lambda L, R: (lambda l, r: True),
    "false": lambda L, R: (lambda l, r: False),
    "l_filter_is_42": lambda L, R: (lambda l, r: None if L[l][1] is None else L[l][1] == 42),
    "r_filter_is_42": lambda L, R: (lambda l, r: None if R[r][1] is None else R[r][1] == 42),
    "l_filter_eq_r_filter": lambda L, R: (lambda l, r: None if L[l][1] is None or R[r][1] is None else L[l][1] == R[r][1]),
}
GRID_TYPES = {"INNER": "inner", "LEFT_OUTER": "left outer", "RIGHT_OUTER": "right outer", "FULL_OUTER": "full outer",
              "LEFT_SEMI": "left semi", "LEFT_ANTI": "left anti", "RIGHT_SEMI": "right semi", "RIGHT_ANTI": "right anti"}


@pytest.mark.parametrize("block", range(len(KAT["residual_grid"]["blocks"])))
def test_residual_filter_grid_kat(block):
    grid = KAT["residual_grid"]
    L, R = grid["left"], grid["right"]
    b = grid["blocks"][block]
    cols = {"l_key": (0, pa.utf8()), "l_filter": (1, pa.int32()), "r_key": (0, pa.utf8()), "r_filter": (1, pa.int32())}
    lkeys = [pa.array([row[cols[n][0]] for row in L], cols[n][1]) for n in b["left_keys"]]
    rkeys = [pa.array([row[cols[n][0]] for row in R], cols[n][1]) for n in b["right_keys"]]
    fn = GRID_FILTERS[b["filter"]](L, R)
    for name, expected in b["expected"].items():
        jt = GRID_TYPES[name]
        pairs = ref_pairs(lkeys, rkeys, jt, residual=fn)
        if jt in ("left semi", "left anti"):
            got = [L[l] for l, _ in pairs]
        elif jt in ("right semi", "right anti"):
            got = [R[r] for _, r in pairs]
        else:
            got = [_gather(L, l) + _gather(R, r) for l, r in pairs]
        assert rows_key(got) == rows_key(expected), (b["filter"], name)
