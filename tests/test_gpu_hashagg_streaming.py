"""Hash aggregates driven as the aggregate node drives them: one state, batches streamed in, the group count growing
between consumes past every reallocation of the state, the consume path changing from batch to batch; the node's loop
over a Grouper; a merge into a destination that grew; a refused shrink.  Every consume checks the kernels it launched
against the restated path plan, every finalize an exact reference over the concatenated input (tests/hashagg_streaming.py)."""
import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import exact_ref as er
from tests import groupings_ref as gr
from tests import hashagg_streaming as hs
from tests.util import SEED

pytestmark = pytest.mark.gpu
SAMPLE = 40  # random groups checked per moment schedule, besides the untouched ones and those one batch touched


def dev(a, ctx):
    return DeviceArray.from_arrow(a, ctx)


def run_schedule(ctx, kind, t, steps, opts_list):
    """one aggregator per option set, all fed the schedule; every step's kernel launches equal the plan's"""
    lib = _cabi.lib()
    aggs = [bc.HashAggregator(kind, t, ctx=ctx, **o) for o in opts_list]
    groups = 0
    for s in steps:
        if s.op == "resize":
            want = hs.plan_resize(kind, groups, s.groups).launches
            for a in aggs:
                before = lib.b2_launch_count()
                a.resize(s.groups)
                assert lib.b2_launch_count() - before == want, (s.name, s.groups)
            groups = s.groups
            continue
        dv, di = s.batch.device(ctx)
        for a, o in zip(aggs, opts_list):
            p = hs.plan_consume(kind, t, groups, s.batch, o.get("skip_nulls", True))
            before = lib.b2_launch_count()
            a.consume(dv, di)
            launched = lib.b2_launch_count() - before
            if p.launches is None:
                assert launched > 0, (s.name, p.path)
            else:
                assert launched == p.launches, (s.name, p.path, o)
    return aggs


def ref_opts(o):
    return {k: v for k, v in o.items() if k in ("skip_nulls", "min_count", "mode")}


def touched_once(steps, groups):
    """groups exactly one batch touched"""
    hits = np.zeros(groups, np.int32)
    for s in steps:
        if s.op == "consume" and s.batch.n:
            hits[np.unique(s.batch.ids)] += 1
    return np.flatnonzero(hits == 1), np.flatnonzero(hits == 0)


def check_moments(kind, t, steps, results, opts_list, rng):
    ids, vals = hs.concat(steps)
    groups = steps[-1].groups
    once, never = touched_once(steps, groups)
    chosen = np.unique(np.concatenate([rng.choice(groups, SAMPLE, replace=False), rng.choice(once, min(20, len(once)), replace=False),
                                       never[:5], never[-5:]]))
    rows = hs.group_rows(ids, vals, chosen)
    for out, o in zip(results, opts_list):
        assert len(out) == groups and out.type == pa.float64()
        ok, raw = er.valid_mask(out), er.raw(out)
        for g in chosen.tolist():
            got = float(raw[g]) if ok[g] else None
            bad = hs.moment_check(kind, t, got, rows.values[g], rows.saw_null[g], **o)
            assert bad is None, (kind, str(t), o, g, bad)


def check_results(kind, t, steps, results, opts_list, seed):
    groups = steps[-1].groups
    if kind in hs.MOMENT_KINDS:
        return check_moments(kind, t, steps, results, opts_list, np.random.default_rng(seed))
    ids, vals = hs.concat(steps)
    _, never = touched_once(steps, groups)
    for out, o in zip(results, opts_list):
        assert len(out) == groups
        if kind in hs.LIST_KINDS:
            gr.assert_same_lists(out, hs.list_reference(kind, ids, vals, groups, **ref_opts(o)))
            continue
        want = hs.reference(kind, ids, vals, groups, **ref_opts(o))
        hs.assert_result(kind, out, want, msg=f"{kind} {t} {o}")
        # the untouched groups hold the identity: the resize fills, nothing else wrote them
        ident = hs.identity(kind, o.get("skip_nulls", True), o.get("min_count", 1))
        tail = out.take(pa.array(never[-1000:]))
        if ident is None:
            assert tail.null_count == len(tail), (kind, o)
        elif isinstance(ident, float):
            assert tail.null_count == 0 and np.isnan(tail.to_numpy(zero_copy_only=False)).all(), (kind, o)
        else:
            assert tail.null_count == 0 and set(tail.to_pylist()) == {ident}, (kind, o)


@pytest.mark.parametrize("kind,t", hs.MATRIX, ids=lambda x: str(x))
def test_streamed_consume(ctx, kind, t):
    opts_list = hs.options(kind)
    seed = hs.seed_of(kind, t)
    steps = hs.schedule(kind, t, seed)
    aggs = run_schedule(ctx, kind, t, steps, opts_list)
    check_results(kind, t, steps, [a.finalize().to_arrow() for a in aggs], opts_list, seed)


@pytest.mark.parametrize("kind,t,opts", hs.BANDED, ids=lambda x: str(x))
def test_streamed_consume_l2_bands(ctx, kind, t, opts):
    seed = hs.seed_of(kind, t, True)
    steps = hs.schedule(kind, t, seed, banded=True)
    aggs = run_schedule(ctx, kind, t, steps, [opts])
    check_results(kind, t, steps, [aggs[0].finalize().to_arrow()], [opts], seed)


# ---- the aggregate node's loop over a Grouper --------------------------------------------------------------------------
UNIVERSE = 5000
# new keys per batch: the group count passes 300, 1024, 1025, 2048, 2049 and UNIVERSE; (key limit, rows)
NODE_BATCHES = [(300, 2 * hs.PRIVATE_MIN_ROWS), (1024, 5000), (1025, 2 * hs.PRIVATE_MIN_ROWS), (1025, 0), (2049, 30_000),
                (2049, 2 * hs.PRIVATE_MIN_ROWS), (UNIVERSE, 60_000)]
NODE_AGGS = [("hash_sum", pa.int64()), ("hash_product", pa.int64()), ("hash_mean", pa.float64()), ("hash_min", pa.int32()),
             ("hash_max", pa.float32()), ("hash_count", pa.string()), ("hash_count_all", None), ("hash_any", pa.bool_()),
             ("hash_all", pa.bool_()), ("hash_count_distinct", pa.string()), ("hash_variance", pa.int16()),
             ("hash_stddev", pa.uint8()), ("hash_skew", pa.float64()), ("hash_kurtosis", pa.int64()),
             ("hash_list", pa.string()), ("hash_distinct", pa.string())]
UNIVERSE_INTS = np.random.default_rng(SEED + 77).choice(np.iinfo(np.int64).max, UNIVERSE, replace=False).astype(np.int64) \
    * np.where(np.arange(UNIVERSE) % 2 == 0, 1, -1)


def key_columns(key_kind, idx):
    """the key columns of universe entries idx"""
    if key_kind == "int64":
        return [pa.array(UNIVERSE_INTS[idx], pa.int64())]
    if key_kind == "utf8":
        return [pa.array([f"key-{int(i) * 7919 % 100003}-{'z' * (int(i) % 5)}" for i in idx], pa.string())]
    return [pa.array((idx % 13).astype(np.int64) - 6, pa.int64()), pa.array([f"s{int(i) // 13}" for i in idx], pa.string())]


def key_rows(batches, rng):
    """universe index per row of each batch; every batch brings the keys up to its limit that earlier ones lacked"""
    out, seen = [], 0
    for limit, n in batches:
        if n == 0:
            out.append(np.zeros(0, np.int64))
            continue
        idx = rng.integers(0, limit, n)
        idx[: limit - seen] = np.arange(seen, limit)
        seen = max(seen, limit)
        out.append(rng.permutation(idx))
    return out


def universe_of(key_kind, uniques):
    """the universe index of each device group, from its unique key"""
    cols = [u.to_arrow().to_pylist() for u in uniques]
    ref = [c.to_pylist() for c in key_columns(key_kind, np.arange(UNIVERSE))]
    table = {tuple(c[i] for c in ref): i for i in range(UNIVERSE)}
    return np.array([table[tuple(c[g] for c in cols)] for g in range(len(cols[0]))], np.int64)


def compare_by_key(kind, t, got, perm, ids, vals, groups, o, msg):
    """got (device groups) against the reference over universe ids; perm[g] = universe index of device group g"""
    order = np.argsort(perm)
    got = got.take(pa.array(order))
    if kind in hs.MOMENT_KINDS:
        check = np.random.default_rng(groups).choice(groups, min(groups, 400), replace=False)
        rows = hs.group_rows(ids, vals, check)
        ok, raw = er.valid_mask(got), er.raw(got)
        for g in check.tolist():
            bad = hs.moment_check(kind, t, float(raw[g]) if ok[g] else None, rows.values[g], rows.saw_null[g], **o)
            assert bad is None, (msg, kind, g, bad)
    elif kind in hs.LIST_KINDS:
        gr.assert_same_lists(got, hs.list_reference(kind, ids, vals, groups, **ref_opts(o)))
    else:
        hs.assert_result(kind, got, hs.reference(kind, ids, vals, groups, **ref_opts(o)), msg=f"{msg} {kind}")


def node_values(kind, t, n, rng):
    return None if t is None else hs.make_values(kind, t, n, rng)


@pytest.mark.parametrize("key_kind", ["int64", "utf8", "int64+utf8"])
def test_node_loop(ctx, key_kind):
    """Grouper.consume, resize(num_groups), consume per batch, then the final resize and finalize, against the reference
    over the concatenation keyed by the universe"""
    rng = np.random.default_rng(SEED + len(key_kind))
    rows = key_rows(NODE_BATCHES, rng)
    vals = {(k, str(t)): [node_values(k, t, len(r), rng) for r in rows] for k, t in NODE_AGGS}
    key_types = [c.type for c in key_columns(key_kind, np.arange(2))]
    g = bc.Grouper(key_types, ctx)
    aggs = {(k, str(t)): bc.HashAggregator(k, t, ctx=ctx) for k, t in NODE_AGGS}
    sizes = []
    for j, r in enumerate(rows):
        ids = g.consume([dev(c, ctx) for c in key_columns(key_kind, r)])
        sizes.append(g.num_groups)
        for (k, ts), a in aggs.items():
            a.resize(g.num_groups)
            v = vals[(k, ts)][j]
            a.consume(None if v is None else dev(v, ctx), ids)
    assert sizes == [300, 1024, 1025, 1025, 2049, 2049, UNIVERSE]
    perm = universe_of(key_kind, g.get_uniques())
    all_ids = np.concatenate(rows).astype(np.uint32)
    for (k, ts), a in aggs.items():
        a.resize(g.num_groups)
        t = dict((str(tt), tt) for _, tt in NODE_AGGS)[ts]
        v = None if t is None else pa.concat_arrays(vals[(k, ts)])
        compare_by_key(k, t, a.finalize().to_arrow(), perm, all_ids, v, UNIVERSE, hs.options(k)[0] if k in hs.MOMENT_KINDS else {},
                       key_kind)


# ---- merge into a destination that grew ------------------------------------------------------------------------------
MERGE_A = [(1000, 2 * hs.PRIVATE_MIN_ROWS), (1000, 4000)]   # A's keys: universe [0, 1000)
MERGE_B = [(3000, 2 * hs.PRIVATE_MIN_ROWS), (3000, 9000)]   # B's keys: [0, 3000), most of them new to A
MERGE_POST = (3600, 7000)                                   # after the merge: [0, 3600)


@pytest.mark.parametrize("kind,t", NODE_AGGS, ids=lambda x: str(x))
def test_merge_into_grown_state(ctx, kind, t):
    """A and B stream their own batches over their own Groupers; B's uniques re-consumed into A's Grouper append B's new
    keys, A grows past its capacity to take them, merges B, consumes once more, finalizes.  Equal, by key, to one
    aggregator over every row in the same order (A's rows, B's, then the last batch)"""
    rng = np.random.default_rng(SEED + hs.seed_of(kind, t) % 1000)
    o = hs.options(kind)[-1]
    ra = key_rows(MERGE_A, rng)
    rb = key_rows(MERGE_B, rng)
    rp = rng.integers(0, MERGE_POST[0], MERGE_POST[1])
    rp[: MERGE_POST[0] - 3000] = np.arange(3000, MERGE_POST[0])
    batches = ra + rb + [rp]
    vals = [node_values(kind, t, len(r), rng) for r in batches]

    def feed(g, agg, j):
        ids = g.consume(dev(key_columns("int64", batches[j])[0], ctx))
        agg.resize(g.num_groups)
        agg.consume(None if vals[j] is None else dev(vals[j], ctx), ids)

    ga, gb, gw = (bc.Grouper([pa.int64()], ctx) for _ in range(3))
    a, b, whole = (bc.HashAggregator(kind, t, ctx=ctx, **o) for _ in range(3))
    for j in range(len(ra)):
        feed(ga, a, j)
    for j in range(len(ra), len(ra) + len(rb)):
        feed(gb, b, j)
    assert ga.num_groups == 1000 and gb.num_groups == 3000
    mapping = ga.consume(gb.get_uniques()[0])
    a.resize(ga.num_groups)
    a.merge(b, mapping)
    feed(ga, a, len(batches) - 1)
    a.resize(ga.num_groups)
    for j in range(len(batches)):
        feed(gw, whole, j)
    assert ga.num_groups == gw.num_groups == MERGE_POST[0]
    ka = ga.get_uniques()[0].to_arrow()
    kw = gw.get_uniques()[0].to_arrow()
    got = a.finalize().to_arrow().take(pa.array(np.argsort(ka.to_numpy())))
    want = whole.finalize().to_arrow().take(pa.array(np.argsort(kw.to_numpy())))
    if kind in hs.LIST_KINDS:
        gr.assert_same_lists(got, want)
    elif kind in hs.MOMENT_KINDS and not hs.is_exact_moments(kind, t):
        # two-pass moments combine partial states with Moments::Merge: the same nulls, each within the bound of the exact
        # statistic
        assert np.array_equal(er.valid_mask(got), er.valid_mask(want))
        perm = np.searchsorted(np.sort(UNIVERSE_INTS[:MERGE_POST[0]]), UNIVERSE_INTS[:MERGE_POST[0]])
        compare_by_key(kind, t, got.take(pa.array(perm)), np.arange(MERGE_POST[0]), np.concatenate(batches).astype(np.uint32),
                       pa.concat_arrays(vals), MERGE_POST[0], o, "merge")
    else:
        hs.assert_result(kind, got, want, msg=f"{kind} {t}")
        ids = np.concatenate(batches).astype(np.uint32)
        v = None if t is None else pa.concat_arrays(vals)
        perm = np.searchsorted(np.sort(UNIVERSE_INTS[:MERGE_POST[0]]), UNIVERSE_INTS[:MERGE_POST[0]])
        compare_by_key(kind, t, got.take(pa.array(perm)), np.arange(MERGE_POST[0]), ids, v, MERGE_POST[0], o, "merge")


# ---- a shrinking resize is refused, and leaves the state as it was -----------------------------------------------------
@pytest.mark.parametrize("kind,t", NODE_AGGS, ids=lambda x: str(x))
def test_shrink_is_refused(ctx, kind, t):
    rng = np.random.default_rng(SEED + 5)
    groups, n = 3000, 20_000
    ids = rng.integers(0, groups - 100, n).astype(np.uint32)
    vals = node_values(kind, t, n, rng)
    o = hs.options(kind)[0]
    a = bc.HashAggregator(kind, t, ctx=ctx, **o)
    a.resize(groups)
    a.consume(None if vals is None else dev(vals, ctx), dev(pa.array(ids), ctx))
    for smaller in (groups - 1, 0):
        with pytest.raises(pa.ArrowInvalid, match="hash aggregate state cannot shrink"):
            a.resize(smaller)
    compare_by_key(kind, t, a.finalize().to_arrow(), np.arange(groups), ids, vals, groups, o, "after a refused shrink")
