"""Exact references for the sort family: array_sort_indices, the multi-key sort, select_k_unstable and the range bins of
the distributed sort's sender side (b2_range_partition / b2_range_split).

The total order is the one sort_indices.cu documents and the reference follows.  A valid value that is not a NaN belongs
to the class "value" and compares by its value: integers as Python ints, floats as Python floats with -0.0 taken as 0.0,
strings by their bytes.  Every NaN (any sign, any payload) belongs to the class "NaN" and every null to the class "null";
within those two classes all rows tie.  The classes come in the order values, NaN, null for "at_end" and null, NaN, values
for "at_start"; "descending" reverses the values only.  Ties keep row order: every sort here is stable.

Nothing here shares the kernels' reasoning (sign flips, IEEE bit tricks, bitwise NOT): the key of a row is a Python tuple
and Python's stable `sorted` orders the rows.  For a few million rows, the `*_np` forms restate the same order with
np.lexsort over (row, canonical value, class); test_sort_edges_oracle.py checks them against the `sorted` forms."""
import math

import numpy as np
import pyarrow as pa

from tests import elementwise_ref as ew
from tests import exact_ref as er

ORDERS = ("ascending", "descending")
PLACEMENTS = ("at_end", "at_start")
VALUE, NAN, NULL = "value", "NaN", "null"
CLASS_RANK = {"at_end": {VALUE: 0, NAN: 1, NULL: 2}, "at_start": {NULL: 0, NAN: 1, VALUE: 2}}


def is_binary(t: pa.DataType) -> bool:
    return pa.types.is_string(t) or pa.types.is_large_string(t) or pa.types.is_binary(t) or pa.types.is_large_binary(t)


def column(arr: pa.Array):
    """(values, valid) of an array: Python ints / floats (null slots hold whatever the buffer holds) or str / bytes"""
    if is_binary(arr.type):
        vals = arr.to_pylist()
        return vals, np.array([v is not None for v in vals], bool)
    return er.raw(arr).tolist(), er.valid_mask(arr)


class _Desc:
    """a str / bytes value whose order is reversed (numbers are negated instead)"""
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = v

    def __lt__(self, other):
        return other.v < self.v

    def __eq__(self, other):
        return self.v == other.v


def value_class(v, ok: bool) -> str:
    if not ok:
        return NULL
    return NAN if isinstance(v, float) and math.isnan(v) else VALUE


def sort_key(v, ok: bool, order: str, placement: str) -> tuple:
    """(class rank, value) of one row; the value part is 0 for NaNs and nulls, so their ties fall through"""
    cls = value_class(v, ok)
    rank = CLASS_RANK[placement][cls]
    if cls != VALUE:
        return rank, 0
    if isinstance(v, float):
        v = v + 0.0                       # -0.0 + 0.0 == +0.0
    if order == "descending":
        v = _Desc(v) if isinstance(v, (str, bytes)) else -v
    return rank, v


def sort_indices_ref(arr: pa.Array, order: str = "ascending", placement: str = "at_end") -> list:
    vals, valid = column(arr)
    keys = [sort_key(v, ok, order, placement) for v, ok in zip(vals, valid.tolist())]
    return sorted(range(len(keys)), key=keys.__getitem__)


def sort_indices_multi_ref(cols, orders, placement: str = "at_end") -> list:
    """lexicographic over the columns (each with its own order), stable"""
    per_col = []
    for arr, order in zip(cols, orders):
        vals, valid = column(arr)
        per_col.append([sort_key(v, ok, order, placement) for v, ok in zip(vals, valid.tolist())])
    keys = list(zip(*per_col))
    return sorted(range(len(cols[0])), key=keys.__getitem__)


def select_k_ref(arr: pa.Array, k: int, order: str = "ascending", placement: str = "at_end") -> list:
    return sort_indices_ref(arr, order, placement)[:k]


def range_key(v, order: str) -> tuple:
    """the range order of partition.cu: a NaN after every value in BOTH orders, -0.0 == +0.0"""
    if isinstance(v, float) and math.isnan(v):
        return 1, 0
    if isinstance(v, float):
        v = v + 0.0
    return 0, (-v if order == "descending" else v)


def range_bin_ref(arr: pa.Array, splitters, order: str = "ascending") -> list:
    """bin of each row: the number of splitters whose key is <= the row's key; a null row goes to len(splitters) + 1"""
    vals, valid = column(arr)
    sk = [range_key(s, order) for s in splitters]
    return [sum(s <= range_key(v, order) for s in sk) if ok else len(sk) + 1 for v, ok in zip(vals, valid.tolist())]


# ---------------------------------------------------------------------------------------------------------------------
# vectorised forms for large inputs (numeric types only)
# ---------------------------------------------------------------------------------------------------------------------
def _canonical(arr: pa.Array, order: str):
    """(canonical values, is NaN, valid): integers in their own dtype (bitwise NOT reverses them exactly), floats with
    NaNs and nulls zeroed and -0.0 made +0.0 (negated for descending)"""
    v, valid = er.raw(arr), er.valid_mask(arr)
    if np.issubdtype(v.dtype, np.floating):
        nan = valid & np.isnan(v)
        c = np.where(nan | ~valid, v.dtype.type(0), v) + v.dtype.type(0)
        if order == "descending":
            c = -c
    else:
        nan = np.zeros(len(v), bool)
        c = np.where(valid, v, v.dtype.type(0))
        if order == "descending":
            c = ~c
    return c, nan, valid


def _class_ranks(nan, valid, placement):
    r = CLASS_RANK[placement]
    return np.where(~valid, r[NULL], np.where(nan, r[NAN], r[VALUE])).astype(np.int8)


def sort_indices_np(arr: pa.Array, order: str = "ascending", placement: str = "at_end") -> np.ndarray:
    c, nan, valid = _canonical(arr, order)
    return np.lexsort((np.arange(len(c)), c, _class_ranks(nan, valid, placement)))


def sort_indices_multi_np(cols, orders, placement: str = "at_end") -> np.ndarray:
    keys = [np.arange(len(cols[0]))]
    for arr, order in reversed(list(zip(cols, orders))):
        c, nan, valid = _canonical(arr, order)
        keys += [c, _class_ranks(nan, valid, placement)]
    return np.lexsort(keys)


def range_bins_np(arr: pa.Array, splitters, order: str = "ascending") -> np.ndarray:
    c, nan, valid = _canonical(arr, order)
    sp = pa.array(np.asarray(splitters, dtype=c.dtype), arr.type)
    sc, snan, _ = _canonical(sp, order)
    bins = np.zeros(len(c), np.int64)
    for s, s_nan in zip(sc, snan):
        bins += nan if s_nan else (nan | (s <= c))     # a NaN row passes every splitter, a NaN splitter only NaN rows
    return np.where(valid, bins, len(sc) + 1)


# ---------------------------------------------------------------------------------------------------------------------
# data: full-range values with the named edge values of the element-wise tests sprinkled in
# ---------------------------------------------------------------------------------------------------------------------
NUMERIC = ew.NUMERIC


def full_range(t: pa.DataType, n: int, rng) -> np.ndarray:
    """n values of t over its whole range: uniform integers, or floats with uniformly random bit patterns (every exponent,
    subnormals, infinities and NaNs of random sign and payload) -- the vectorised form of test_gpu_elementwise_edges'
    random_values, for millions of rows"""
    dt = ew.np_dtype(t)
    if pa.types.is_integer(t):
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
    u = er.UINT_OF_WIDTH[dt.itemsize]
    return rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(dt)


def edge_pool(t: pa.DataType) -> np.ndarray:
    """the named edge values of t (elementwise_ref.edges) and, for floats, every special bit pattern of
    exact_ref (NaNs of both signs and several payloads, the signalling one included, +-0, +-inf, the least subnormal)"""
    dt = ew.np_dtype(t)
    if pa.types.is_integer(t):
        return np.array(ew.edges(t), dtype=object).astype(dt)
    return np.concatenate([np.array(ew.edges(t), np.float64).astype(dt), er.special_values(dt)])


def edge_values(t: pa.DataType, n: int, rng, edge_p: float = 0.4) -> np.ndarray:
    """full-range values where a fraction edge_p of the rows holds an edge value (so edges tie with each other)"""
    v = full_range(t, n, rng)
    pick = rng.random(n) < edge_p
    pool = edge_pool(t)
    v[pick] = pool[rng.integers(0, len(pool), int(pick.sum()))]
    return v


def to_arrow(t: pa.DataType, v: np.ndarray, valid=None, offset: int = 0) -> pa.Array:
    """an Arrow array of t over exactly these bits (never through Python floats), sliced at `offset`: the first `offset`
    rows of v are dropped"""
    v = np.ascontiguousarray(v, dtype=ew.np_dtype(t))
    if valid is None or np.all(valid):
        bufs, nc = [None, pa.py_buffer(v.tobytes())], 0
    else:
        valid = np.asarray(valid, bool)
        bufs, nc = [pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()), pa.py_buffer(v.tobytes())], int((~valid).sum())
    arr = pa.Array.from_buffers(t, len(v), bufs, null_count=nc)
    return arr.slice(offset) if offset else arr


def edge_array(t: pa.DataType, n: int, rng, null_p: float = 0.1, offset: int = 0, edge_p: float = 0.4) -> pa.Array:
    m = n + offset
    return to_arrow(t, edge_values(t, m, rng, edge_p), rng.random(m) >= null_p, offset)


STRINGS = ["", "a", "a\x00", "ab", "b", "é", "été", "zz", "\U0001F600", "A"]


def multi_columns(n, rng) -> dict:
    """key columns for the multi-key sorts, each sliced at its own offset: float64 NaN payloads, +-0 and +-inf (ties that
    must fall through to the next key), int64 extremes, short utf8 strings, full-range uint8 and float32 edge values"""
    f = edge_pool(pa.float64())
    f = f[np.isnan(f) | (f == 0) | np.isinf(f)]                      # NaN payloads, +-0 and +-inf: many ties
    i = np.array([-(1 << 63), -1, 0, 1, (1 << 63) - 1], np.int64)
    return {
        "f": to_arrow(pa.float64(), f[rng.integers(0, len(f), n + 1)], rng.random(n + 1) > 0.1, 1),
        "i": to_arrow(pa.int64(), i[rng.integers(0, len(i), n + 2)], rng.random(n + 2) > 0.1, 2),
        "s": pa.array([STRINGS[j] if j < len(STRINGS) else None for j in rng.integers(0, len(STRINGS) + 1, n + 3)],
                      pa.utf8()).slice(3),
        "u": to_arrow(pa.uint8(), full_range(pa.uint8(), n, rng), rng.random(n) > 0.05),
        "g": to_arrow(pa.float32(), edge_values(pa.float32(), n + 5, rng, 0.9), rng.random(n + 5) > 0.2, 5),
    }


MULTI_KEYS = [
    [("f", "ascending")],
    [("s", "descending")],
    [("f", "descending"), ("i", "ascending")],
    [("s", "ascending"), ("f", "ascending"), ("u", "descending")],
    [("i", "descending"), ("s", "descending"), ("g", "ascending"), ("u", "ascending")],
    [("g", "descending"), ("f", "ascending"), ("i", "ascending"), ("u", "descending")],
]
