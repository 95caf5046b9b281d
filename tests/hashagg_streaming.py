"""A hash aggregate fed as the aggregate node feeds it: one state, a stream of batches, the group count growing between
consumes (b200_acero.cc ConsumeDevice: Grouper::Consume, resize(num_groups), consume; MaybeFinish: resize, finalize).

Schedule.  A seeded list of resize / consume steps for one (kind, value type).  The group count starts below the
state's minimum capacity and grows to exactly it, one past it, to twice it, one past that and to millions, so every
reallocation of the state happens with live state.  The batches take each consume path of the kind, in an order where
a path adds into state another path wrote (private kernel, then atomics, then the private kernel again, ...).  After
the large growth a batch touches only old ids, so the new groups keep the identity until a later batch reaches them;
a tail of groups is never touched.  There is a zero-length batch, a batch cut from a longer device array at an odd row
offset (null_count unknown, as FlushRun passes runs), a batch whose validity buffer is present without nulls, an
all-null batch, a batch of special floats (NaN payloads, +-inf, +-0, denormals) on groups no other batch touches, a
repeated resize and the final resize before finalize.

Path plan.  launch_consume / b2_hashagg_consume / b2_hashagg_resize (hash_aggregate.cu) and run_pass / consume_typed /
moments_resize (hash_moments.cu) restated: for each step the path taken and the kernels launched.  The thresholds are
read from the sources; hash_sum's dense decision is packed_regimes.byid_plan.

References.  Over the concatenated input, exact: integer sums and products wrap mod 2^64 in any order; float values are
dyadic (sums exact in any order) or +-2^k (products exact); hash_mean over integers keeps every partial sum below
2^53, so the mean is the exact sum over the count, rounded once."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pyarrow as pa

from oracle import arrow_oracle as ora
from tests import exact_ref as er
from tests import groupings_ref as gr
from tests import moments_ref as mr
from tests import packed_regimes as P

_HASHAGG = P._read("hash_aggregate.cu")
_MOMENTS = P._read("hash_moments.cu")

# ---- thresholds, from the sources ----------------------------------------------------------------------------------
K_PRIVATE_MAX_GROUPS = P.K_PRIVATE_MAX_GROUPS
HASHAGG_BAND_BYTES = P.HASHAGG_BAND_BYTES
HASHAGG_BAND_MIN_ROWS = P.HASHAGG_BAND_MIN_ROWS
PRIVATE_MIN_ROWS = 1 << int(P._find(_HASHAGG, r"a->num_groups <= kPrivateMaxGroups && n >= \(1 << (\d+)\) && a->kind").group(1))
assert PRIVATE_MIN_ROWS == 1 << int(P._find(_HASHAGG, r"few_groups = a->num_groups <= kPrivateMaxGroups && n >= \(1 << (\d+)\);").group(1))
# state bytes per group of one band: reduced + counts, or counts alone for hash_count
_m = P._find(_HASHAGG, r"hashagg_band_bytes\(\) / \(two_arrays \? (\d+) : (\d+)\);")
BAND_BYTES_PER_GROUP, COUNT_BAND_BYTES_PER_GROUP = int(_m.group(1)), int(_m.group(2))
# the smallest capacity of a state; beyond it the next power of two
MIN_CAP = int(P._find(_HASHAGG, r"next_pow2\(num_groups < (\d+) \? \1 : num_groups\)").group(1))
assert MIN_CAP == int(P._find(_MOMENTS, r"next_pow2\(num_groups < (\d+) \? \1 : num_groups\)").group(1))
K_MOMENT_PRIVATE_GROUPS = int(P._find(_MOMENTS, r"constexpr int kMomentPrivateGroups = (\d+);").group(1))
MOMENT_PRIVATE_MIN_ROWS = 1 << int(P._find(_MOMENTS, r"m->num_groups <= kMomentPrivateGroups && n >= \(1 << (\d+)\)").group(1))
MOMENT_BAND_MIN_ROWS = 1 << int(P._find(_MOMENTS, r"if \(bands < 1 \|\| n < \(1 << (\d+)\)\) bands = 1;").group(1))
_m = P._find(_MOMENTS, r"constexpr int kStatePlanes = (\d+), kBatchPlanes = (\d+)")
MOMENT_STATE_PLANES = int(_m.group(1))

NUMERIC_KINDS = ("hash_sum", "hash_product", "hash_mean", "hash_min", "hash_max")
MOMENT_KINDS = ("hash_variance", "hash_stddev", "hash_skew", "hash_kurtosis")
LIST_KINDS = ("hash_list", "hash_distinct")
PAIR_KINDS = ("hash_count_distinct", "hash_distinct")
LEVEL = {"hash_variance": 2, "hash_stddev": 2, "hash_skew": 3, "hash_kurtosis": 4}
NARROW_INTS = (pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32())

# millions of groups: enough for hash_count's state (8 bytes a group) to take two L2 bands
G_BIG = HASHAGG_BAND_BYTES // COUNT_BAND_BYTES_PER_GROUP + 100_003


def is_numeric(t) -> bool:
    return t is not None and (pa.types.is_integer(t) or pa.types.is_floating(t))


def is_exact_moments(kind, t) -> bool:
    return kind in MOMENT_KINDS and LEVEL[kind] == 2 and t in NARROW_INTS


def _bands(groups: int, n: int, bytes_per_group: int, min_rows: int) -> int:
    band_groups = HASHAGG_BAND_BYTES // bytes_per_group
    b = -(-groups // band_groups)
    return 1 if b < 1 or n < min_rows else b


def _banded(b: int) -> str:
    return f"banded({b})" if b > 1 else "atomic"


def path_family(path: str) -> str:
    """banded(k) -> banded"""
    return path.split("(")[0]


# ---- the schedule ------------------------------------------------------------------------------------------------
@dataclass
class Batch:
    """one consume: `ids` / `values` are the rows the kernel sees (values None for hash_count_all).  layout:
    plain, sliced (rows [offset, offset + n) of the longer `parent_*` arrays), valid_no_nulls (a validity buffer with every
    bit set, null_count unknown), all_null, empty, special"""
    ids: np.ndarray
    values: Optional[pa.Array]
    layout: str = "plain"
    offset: int = 0
    parent_ids: Optional[np.ndarray] = None
    parent_values: Optional[pa.Array] = None

    @property
    def n(self) -> int:
        return len(self.ids)

    @property
    def null_count(self) -> int:
        """the null_count the kernel is handed"""
        if self.values is None:
            return 0
        if self.layout == "valid_no_nulls":
            return -1
        if self.layout == "sliced":
            return -1 if self.parent_values.null_count else 0
        return self.values.null_count

    def valid(self) -> np.ndarray:
        return np.ones(self.n, bool) if self.values is None else er.valid_mask(self.values)

    def device(self, ctx):
        """(values, ids) as DeviceArrays in the batch's layout"""
        from arrow_b200 import DeviceArray
        if self.layout == "sliced":
            di = DeviceArray.from_arrow(pa.array(self.parent_ids, pa.uint32()), ctx).slice(self.offset, self.n)
            dv = None if self.values is None else DeviceArray.from_arrow(self.parent_values, ctx).slice(self.offset, self.n)
            return dv, di
        di = DeviceArray.from_arrow(pa.array(self.ids, pa.uint32()), ctx)
        if self.values is None:
            return None, di
        if self.layout == "valid_no_nulls":
            ones = pa.py_buffer(np.packbits(np.ones(self.n, bool), bitorder="little").tobytes())
            arr = pa.Array.from_buffers(self.values.type, self.n, [ones] + self.values.buffers()[1:], null_count=0)
            dv = DeviceArray.from_arrow(arr, ctx)
            dv.null_count = -1
            return dv, di
        return DeviceArray.from_arrow(self.values, ctx), di


@dataclass
class Step:
    op: str  # resize / consume
    groups: int  # the state's group count after the step
    batch: Optional[Batch] = None
    name: str = ""


@dataclass(frozen=True)
class Sizes:
    first: int = 300                            # the first resize, below MIN_CAP
    big: int = G_BIG                            # millions of groups
    private_rows: int = 2 * PRIVATE_MIN_ROWS    # the private kernel's batches
    small_rows: int = 5000                      # below PRIVATE_MIN_ROWS: atomics at any group count
    atomic_rows: int = 30_000
    dense_rows: int = P.DENSE_MIN_ROWS + 7      # hash_sum's dense packed path by id
    band_rows: int = HASHAGG_BAND_MIN_ROWS + 5  # the L2 bands
    late_rows: int = 1 << 17                    # reaches the groups added by the large growth
    null_span: int = 50_000                     # groups the all-null batch touches
    special_groups: int = 1000
    tail: int = 100_000                         # groups no batch touches


FULL = Sizes()
# the same steps at sizes pyarrow and Python references handle in a moment (the paths are not the point there)
SMALL = Sizes(first=30, big=6000, private_rows=700, small_rows=300, atomic_rows=500, dense_rows=900, band_rows=1500,
              late_rows=800, null_span=200, special_groups=60, tail=300)


def _mask(rng, n, p=0.1):
    return rng.random(n) < p


def _ints(t, n, rng, kind, role, sizes):
    dt = np.dtype(t.to_pandas_dtype())
    info = np.iinfo(dt)
    if kind == "hash_mean" and dt.itemsize == 8:
        # every partial sum stays below 2^53: the mean is exact_sum / count, rounded once
        lo, hi = (-(1 << 31), 1 << 31) if dt.kind == "i" else (0, 1 << 32)
        return rng.integers(lo, hi, n).astype(dt)
    if kind in MOMENT_KINDS and dt.itemsize == 8:
        return (10**12 + rng.integers(-10**4, 10**4, n)).astype(dt)
    if role == "dense" and dt.itemsize == 8:
        # a narrow window at the top of the type: hash_sum's dense path takes 64-bit values whose sampled range fits
        return (info.max - rng.integers(0, 1 << 15, n).astype(np.uint64)).astype(dt)
    v = rng.integers(int(info.min), int(info.max), n, dtype=dt, endpoint=True)
    if kind == "hash_product":
        v |= dt.type(1)  # odd factors: a product of many rows does not collapse to 0 mod 2^64
    salt = rng.random(n) < 1 / 64
    v[salt] = rng.choice(np.array([info.min, info.max], dt), int(salt.sum()))
    return v


def _floats(t, n, rng, kind):
    dt = np.dtype(t.to_pandas_dtype())
    if kind == "hash_product":
        return rng.choice(np.array([0.5, 1, 2, -0.5, -1, -2], dt), n)  # +-2^k: products exact
    if kind in MOMENT_KINDS:
        return rng.normal(1e3, 1.0, n).astype(dt)
    return (rng.integers(-(1 << 19), 1 << 19, n) / 16.0).astype(dt)  # dyadic: every partial sum exact in double


WORDS = np.array(["", "a", "bb", "ccc", "héllo", "x" * 40] + [f"w{i}" for i in range(40)], dtype=object)


def make_values(kind, t, n, rng, role="plain", sizes=FULL, null_p=0.1) -> Optional[pa.Array]:
    if t is None:
        return None
    mask = np.ones(n, bool) if role == "all_null" else (_mask(rng, n, null_p) if role not in ("valid_no_nulls",) else None)
    if pa.types.is_boolean(t):
        return pa.array(rng.random(n) < 0.8, pa.bool_(), mask=mask)
    if pa.types.is_string(t):
        return pa.array(rng.choice(WORDS, n).tolist(), pa.string(), mask=mask)
    v = _floats(t, n, rng, kind) if pa.types.is_floating(t) else _ints(t, n, rng, kind, role, sizes)
    return pa.array(v, t, mask=mask)


def _batch(kind, t, ids, rng, role="plain", sizes=FULL) -> Batch:
    ids = np.asarray(ids, np.uint32)
    n = len(ids)
    if kind == "hash_count_all":
        t = None
    if role == "sliced":
        pre, post = 7, 5  # an odd row offset: bit offset 7 of the validity and boolean data
        pids = np.concatenate([rng.integers(0, max(int(ids.max()) + 1 if n else 1, 1), pre).astype(np.uint32), ids,
                               np.zeros(post, np.uint32)])
        pv = None
        if t is not None:
            pv = make_values(kind, t, pre + n + post, rng, "plain", sizes, null_p=0.1)
            if pv.null_count == 0:
                pv = pa.array(pv.to_pylist()[:-1] + [None], t)
        return Batch(ids, None if pv is None else pv.slice(pre, n), "sliced", pre, pids, pv)
    if role == "special" and t is not None and pa.types.is_floating(t) and kind in NUMERIC_KINDS:
        local, vals = er.special_float_groups(t.to_pandas_dtype(), sizes.special_groups, n, int(rng.integers(1 << 30)))
        return Batch(ids.min() + local if n else ids, vals, "special")
    return Batch(ids, make_values(kind, t, n, rng, role, sizes), role)


def schedule(kind, t, seed: int, sizes: Sizes = FULL, banded=False) -> list:
    """the steps for one aggregator of `kind` over values of type `t` (None for hash_count_all)"""
    rng = np.random.default_rng(seed)
    cap = MIN_CAP
    s_lo = sizes.big - sizes.tail - sizes.special_groups  # the special batch's groups: no other batch touches them
    null_hi = min(2 * cap + 1 + sizes.null_span, s_lo)
    rows = lambda lo, hi, n: rng.integers(lo, hi, n).astype(np.uint32)  # noqa: E731
    b = lambda ids, role="plain": _batch(kind, t, ids, rng, role, sizes)  # noqa: E731
    dense_n = sizes.dense_rows if kind == "hash_sum" else sizes.atomic_rows
    steps = [
        Step("resize", sizes.first, name="first resize, below the minimum capacity"),
        # groups sizes.first - 10 .. sizes.first - 1 wait for a later batch
        Step("consume", sizes.first, b(rows(0, sizes.first - 10, sizes.private_rows)), "private kernel"),
        Step("resize", cap, name="exactly the capacity"),
        Step("consume", cap, b(rows(0, cap, sizes.small_rows), "valid_no_nulls"), "atomics into the private kernel's state"),
        Step("resize", cap + 1, name="one past the capacity: reallocation"),
        Step("consume", cap + 1, b(rows(0, cap + 1, sizes.private_rows), "sliced"), "private kernel into atomic state"),
        Step("resize", 2 * cap, name="twice the capacity"),
        Step("resize", 2 * cap, name="the same count again"),
        Step("consume", 2 * cap, b(np.zeros(0, np.uint32)), "zero rows"),
        Step("resize", 2 * cap + 1, name="one past: reallocation"),
        Step("consume", 2 * cap + 1, b(rows(0, 2 * cap + 1, dense_n), "dense"), "past the private kernel"),
        Step("resize", sizes.big, name="millions of groups: reallocation"),
        Step("consume", sizes.big, b(rows(0, 2 * cap + 1, sizes.small_rows)), "old ids only"),
        Step("consume", sizes.big, b(rows(2 * cap + 1, null_hi, sizes.small_rows), "all_null"), "every row null"),
        Step("consume", sizes.big, b(s_lo + (np.arange(4 * sizes.special_groups) % sizes.special_groups).astype(np.uint32),
                                     "special"), "special floats on groups of their own"),
    ]
    if banded:
        steps.append(Step("consume", sizes.big, b(rows(0, s_lo, sizes.band_rows)), "L2 bands"))
    steps += [
        Step("consume", sizes.big, b(rows(0, s_lo, sizes.late_rows)), "reaches the new groups"),
        Step("resize", sizes.big, name="the final resize before finalize"),
    ]
    return steps


def concat(steps):
    """(ids, values) of every consumed row in consume order"""
    batches = [s.batch for s in steps if s.op == "consume"]
    ids = np.concatenate([b.ids for b in batches]).astype(np.uint32)
    vals = [b.values for b in batches]
    return ids, (None if vals[0] is None else pa.concat_arrays(vals))


# ---- the path plan -----------------------------------------------------------------------------------------------
@dataclass
class StepPlan:
    path: str
    launches: Optional[int]  # None: the pair Grouper's own kernels (at least one)


def plan_resize(kind, old: int, new: int) -> StepPlan:
    """b2_hashagg_resize: the identity fill (hashagg_fill_kernel / moments_zero_kernel) of the added groups; the pair
    Grouper and the list state keep only the count"""
    if kind in PAIR_KINDS or kind == "hash_list":
        return StepPlan("resize", 0)
    return StepPlan("resize", 1 if new > old else 0)


def _moment_plan(kind, t, groups, n) -> StepPlan:
    level = LEVEL[kind]

    def run_pass(planes, extra):
        if groups <= K_MOMENT_PRIVATE_GROUPS and n >= MOMENT_PRIVATE_MIN_ROWS:
            return "private", 1
        b = _bands(groups, n, 8 * (planes + extra), MOMENT_BAND_MIN_ROWS)
        return _banded(b), b

    if is_exact_moments(kind, t):
        return StepPlan(*run_pass(MOMENT_STATE_PLANES, 0))
    p1, k1 = run_pass(2 if pa.types.is_floating(t) else 3, 0)  # count, sum (double, or two 64-bit limbs)
    _, k2 = run_pass(level - 1, 1)                               # the central moments, reading the means
    return StepPlan(p1, k1 + 1 + k2 + 1)                          # + moments_means_kernel + moments_merge_batch_kernel


def plan_consume(kind, t, groups: int, batch: Batch, skip_nulls=True) -> StepPlan:
    n = batch.n
    if n == 0:
        return StepPlan("empty", 0)
    if kind in MOMENT_KINDS:
        return _moment_plan(kind, t, groups, n)
    if kind == "hash_list":
        # the validity bits, then the boolean data bits or the rebased string offsets (fixed width: copies only)
        return StepPlan("list", 1 + (1 if pa.types.is_boolean(t) or pa.types.is_string(t) else 0))
    if kind in PAIR_KINDS:
        return StepPlan("pairs", None)
    few = groups <= K_PRIVATE_MAX_GROUPS and n >= PRIVATE_MIN_ROWS
    if kind == "hash_count_all":
        return StepPlan("private" if few else "countall", 1)
    if kind == "hash_count" and not is_numeric(t):
        return StepPlan("private" if few else "atomic", 1)
    if kind in ("hash_any", "hash_all"):
        return StepPlan("bool", 1)
    if few and kind != "hash_product":
        return StepPlan("private", 1)
    per_group = COUNT_BAND_BYTES_PER_GROUP if kind == "hash_count" else BAND_BYTES_PER_GROUP
    bands = _bands(groups, n, per_group, HASHAGG_BAND_MIN_ROWS)
    if kind == "hash_sum" and pa.types.is_integer(t):
        if not (skip_nulls or batch.null_count == 0):
            return StepPlan(_banded(bands), bands)  # the dense path keeps no has-null flags
        vals = er.raw(batch.values)
        p = P.byid_plan(batch.ids, groups, vals, batch.valid(), skip_nulls=True)
        launches = p.launches(t.bit_width // 8, n, groups)
        return StepPlan("dense" if p.dense is not None else _banded(bands), launches)
    return StepPlan(_banded(bands), bands)


def kind_paths(kind, t) -> set:
    """every path family a consume of `kind` over `t` can take"""
    if kind in MOMENT_KINDS:
        return {"private", "atomic", "banded"}
    if kind == "hash_list":
        return {"list"}
    if kind in PAIR_KINDS:
        return {"pairs"}
    if kind == "hash_count_all":
        return {"private", "countall"}
    if kind in ("hash_any", "hash_all"):
        return {"bool"}
    if kind == "hash_count" and not is_numeric(t):
        return {"private", "atomic"}
    paths = {"atomic", "banded"} | (set() if kind == "hash_product" else {"private"})
    return paths | ({"dense"} if kind == "hash_sum" and pa.types.is_integer(t) else set())


def planned_paths(kind, t, steps, skip_nulls=True) -> list:
    """(step, StepPlan) for every step"""
    out, groups = [], 0
    for s in steps:
        if s.op == "resize":
            out.append((s, plan_resize(kind, groups, s.groups)))
            groups = max(groups, s.groups)
        else:
            out.append((s, plan_consume(kind, t, groups, s.batch, skip_nulls)))
    return out


# ---- references ----------------------------------------------------------------------------------------------------
def reference(kind, ids, vals, groups, skip_nulls=True, min_count=1, mode="only_valid") -> pa.Array:
    """finalize of `kind` (not a list, not a moment) over the concatenated rows"""
    ids = np.asarray(ids, np.int64)
    if kind == "hash_count_all":
        return pa.array(np.bincount(ids, minlength=groups).astype(np.int64))
    if kind == "hash_count":
        ok = er.valid_mask(vals)
        sel = ok if mode == "only_valid" else (~ok if mode == "only_null" else np.ones(len(ids), bool))
        return pa.array(np.bincount(ids[sel], minlength=groups).astype(np.int64))
    if kind == "hash_count_distinct":
        if pa.types.is_string(vals.type) or pa.types.is_binary(vals.type):
            vals = vals.dictionary_encode().indices  # the same distinct values, as fixed-width codes
        return pa.array(er.count_distinct(ids, vals, groups, mode))
    return ora.hash_aggregate(kind, vals, pa.array(ids.astype(np.uint32)), groups, skip_nulls=skip_nulls,
                              min_count=min_count)


def list_reference(kind, ids, vals, groups, mode="only_valid") -> pa.Array:
    if kind == "hash_list":
        return gr.hash_list(vals, pa.array(ids, pa.uint32()), groups)
    return gr.hash_distinct(vals, ids, groups, mode)


def assert_result(kind, got: pa.Array, want: pa.Array, msg=""):
    """er.assert_same (bits; -0.0 == +0.0 for min / max), booleans by validity and value"""
    if pa.types.is_boolean(want.type):
        gv, wv = er.valid_mask(got), er.valid_mask(want)
        assert got.type == want.type and np.array_equal(gv, wv), msg
        g, w = np.asarray(got.fill_null(False)), np.asarray(want.fill_null(False))
        bad = np.flatnonzero(gv & (g != w))
        assert len(bad) == 0, f"{msg}: {len(bad)} differ, at {bad[:5].tolist()}"
        return
    er.assert_same(got, want, zeros_equal=kind in ("hash_min", "hash_max"), msg=msg)


def identity(kind, skip_nulls=True, min_count=1):
    """the result of a group that no batch touched (None: null)"""
    if kind in ("hash_sum", "hash_product", "hash_any", "hash_all"):
        return {"hash_sum": 0, "hash_product": 1, "hash_any": False, "hash_all": True}[kind] if min_count == 0 else None
    if kind == "hash_mean":
        return math.nan if min_count == 0 else None
    if kind in ("hash_min", "hash_max") or kind in MOMENT_KINDS:
        return None
    if kind in LIST_KINDS:
        return []
    return 0  # counts, hash_count_distinct


@dataclass
class GroupRows:
    """the valid values and the saw-a-null flag of chosen groups over the concatenated rows"""
    values: dict = field(default_factory=dict)
    saw_null: dict = field(default_factory=dict)


def group_rows(ids, vals: pa.Array, chosen) -> GroupRows:
    ok = er.valid_mask(vals)
    raw = er.raw(vals)
    order = np.argsort(ids, kind="stable")
    sids = ids[order]
    out = GroupRows()
    for g in chosen:
        lo, hi = np.searchsorted(sids, g), np.searchsorted(sids, g, side="right")
        rows = order[lo:hi]
        out.values[int(g)] = raw[rows][ok[rows]]
        out.saw_null[int(g)] = bool((~ok[rows]).any())
    return out


def moment_expected(kind, t, xs: np.ndarray, saw_null: bool, ddof=0, biased=True, skip_nulls=True, min_count=0):
    """the statistic of the valid values xs: None when it is null, else (value, tolerance).  Exact on the exact path
    (8- to 32-bit integers, variance / stddev: a Fraction rounded once); on the two-pass path the exact statistic and
    moments_ref.tolerance; without spread 0 for variance / stddev and 0 / 0 for skew and kurtosis"""
    fn = kind[len("hash_"):]
    n = len(xs)
    if mr.is_null(fn, n, saw_null, ddof, skip_nulls, min_count, biased):
        return None
    if is_exact_moments(kind, t):
        ints = [int(v) for v in xs]
        v = float(mr.Fraction(n * sum(x * x for x in ints) - sum(ints) ** 2, n * (n - ddof)))
        return (math.sqrt(v) if fn == "stddev" else v), 0.0
    if len(np.unique(xs)) < 2:
        return (0.0 if fn in ("variance", "stddev") else math.nan), 0.0
    exact = mr.exact_statistic(fn, xs, ddof, biased)
    # the relative bound, or the absolute one where it is wider: kurtosis is n m4 / m2^2 - 3, and near 0 the subtraction
    # magnifies the moments' relative error (few values per group, data offset far from 0)
    rel = mr.tolerance(fn, xs)
    tol = mr.tolerance_abs(fn, xs)
    return exact, (max(rel * abs(exact), tol) if exact != 0 and math.isfinite(rel) else tol)


def moment_check(kind, t, got: Optional[float], xs: np.ndarray, saw_null: bool, slack=0.0, **opts) -> Optional[str]:
    """None when `got` is the statistic of xs (moment_expected, its tolerance widened by slack * |value|); else what
    differs"""
    want = moment_expected(kind, t, xs, saw_null, **opts)
    if want is None or got is None:
        return None if want is None and got is None else f"got {got!r}, want {want!r}"
    v, tol = want
    if math.isnan(v) or math.isnan(got):
        return None if math.isnan(v) and math.isnan(got) else f"got {got!r}, want {v!r}"
    return None if abs(got - v) <= tol + slack * abs(v) else f"got {got!r}, exact {v!r}, tolerance {tol!r}"


# ---- what the device tests run ---------------------------------------------------------------------------------------
NUMERIC_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64(),
                 pa.float32(), pa.float64()]
SCALAR_OPTIONS = [dict(skip_nulls=s, min_count=m) for s in (True, False) for m in (0, 1, 3)]
MODES = [dict(mode=m) for m in ("only_valid", "only_null", "all")]
MOMENT_OPTIONS = {
    2: [dict(ddof=0), dict(ddof=1, skip_nulls=False), dict(ddof=2, min_count=3)],
    3: [dict(biased=True), dict(biased=False, skip_nulls=False), dict(biased=False, min_count=3)],
}


def options(kind) -> list:
    if kind in MOMENT_KINDS:
        return MOMENT_OPTIONS[2 if LEVEL[kind] == 2 else 3]
    if kind in ("hash_count", "hash_count_distinct", "hash_distinct"):
        return MODES
    if kind in ("hash_count_all", "hash_list"):
        return [{}]
    return SCALAR_OPTIONS


# (kind, value type) streamed at the smaller sizes, every option set on its own aggregator
MATRIX = ([(k, t) for k in NUMERIC_KINDS + MOMENT_KINDS for t in NUMERIC_TYPES]
          + [("hash_count", pa.string()), ("hash_count", pa.int64()), ("hash_count_all", None),
             ("hash_any", pa.bool_()), ("hash_all", pa.bool_()), ("hash_count_distinct", pa.string()),
             ("hash_distinct", pa.string()), ("hash_list", pa.string())])
# (kind, value type, option set) streamed with the L2-banded batch as well
BANDED = ([(k, t, options(k)[1]) for k in NUMERIC_KINDS for t in (pa.int64(), pa.uint8(), pa.float64())]
          + [("hash_count", pa.int64(), MODES[2]), ("hash_any", pa.bool_(), SCALAR_OPTIONS[3]),
             ("hash_all", pa.bool_(), SCALAR_OPTIONS[1]), ("hash_variance", pa.uint8(), MOMENT_OPTIONS[2][1]),
             ("hash_stddev", pa.int64(), MOMENT_OPTIONS[2][0]), ("hash_skew", pa.float64(), MOMENT_OPTIONS[3][1]),
             ("hash_kurtosis", pa.int32(), MOMENT_OPTIONS[3][0])])


def seed_of(kind, t, banded=False) -> int:
    import zlib
    return zlib.crc32(f"{kind}/{t}/{banded}".encode())
