"""CPU: the streamed hash aggregates' references (tests/hashagg_streaming.py) against the reference binary (pyarrow's
group_by) over the concatenated batches of small schedules, the identities of groups no batch touched, and the path plan:
its constants parse, and the schedules the device tests run reach every consume path of every kind and every
reallocation of the state."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from tests import exact_ref as er
from tests import groupings_ref as gr
from tests import hashagg_streaming as hs

PA_NAME = {"hash_sum": "sum", "hash_product": "product", "hash_mean": "mean", "hash_min": "min", "hash_max": "max",
           "hash_count": "count", "hash_any": "any", "hash_all": "all", "hash_count_distinct": "count_distinct",
           "hash_variance": "variance", "hash_stddev": "stddev", "hash_skew": "skew", "hash_kurtosis": "kurtosis",
           "hash_list": "list", "hash_distinct": "distinct"}
ORACLE_MATRIX = ([(k, t) for k in hs.NUMERIC_KINDS for t in (pa.int8(), pa.uint64(), pa.int64(), pa.float32(), pa.float64())]
                 + [(k, t) for k in hs.MOMENT_KINDS for t in (pa.int16(), pa.uint32(), pa.int64(), pa.float64())]
                 + [(k, t) for k, t in hs.MATRIX if k not in hs.NUMERIC_KINDS + hs.MOMENT_KINDS])


def pa_options(kind, o):
    if kind in ("hash_count", "hash_count_distinct", "hash_distinct"):
        return pc.CountOptions(o["mode"])
    if kind in ("hash_variance", "hash_stddev"):
        return pc.VarianceOptions(ddof=o.get("ddof", 0), skip_nulls=o.get("skip_nulls", True), min_count=o.get("min_count", 0))
    if kind in ("hash_skew", "hash_kurtosis"):
        return pc.SkewOptions(skip_nulls=o.get("skip_nulls", True), biased=o.get("biased", True), min_count=o.get("min_count", 0))
    if kind == "hash_list":
        return None
    return pc.ScalarAggregateOptions(skip_nulls=o["skip_nulls"], min_count=o["min_count"])


def acero(kind, ids, vals, o):
    """(group ids present, result per present group) from pyarrow's group_by over the concatenated rows"""
    import pyarrow.acero  # noqa: F401
    if kind == "hash_count_all":
        t = pa.table({"g": pa.array(ids, pa.uint32())}).group_by("g", use_threads=False).aggregate([([], "count_all")])
        col = "count_all"
    else:
        t = pa.table({"g": pa.array(ids, pa.uint32()), "v": vals}).group_by("g", use_threads=False).aggregate(
            [("v", PA_NAME[kind], pa_options(kind, o))])
        col = f"v_{PA_NAME[kind]}"
    return t["g"].to_numpy().astype(np.int64), t[col].combine_chunks()


@pytest.mark.parametrize("kind,t", ORACLE_MATRIX, ids=lambda x: str(x))
def test_references_vs_reference_binary(kind, t):
    steps = hs.schedule(kind, t, hs.seed_of(kind, t), hs.SMALL)
    ids, vals = hs.concat(steps)
    groups = steps[-1].groups
    untouched = np.setdiff1d(np.arange(groups), ids)
    assert len(untouched) >= hs.SMALL.tail
    for o in hs.options(kind):
        present, want = acero(kind, ids, vals, o)
        if kind in hs.MOMENT_KINDS:
            rows = hs.group_rows(ids, vals, np.arange(groups))
            w_ok, w_raw = er.valid_mask(want), want.to_numpy(zero_copy_only=False)
            for j, g in enumerate(present.tolist()):
                # the reference rounds the exact path's statistic twice, the device once
                bad = hs.moment_check(kind, t, float(w_raw[j]) if w_ok[j] else None, rows.values[g], rows.saw_null[g],
                                      slack=1e-12 if hs.is_exact_moments(kind, t) else 0.0, **o)
                assert bad is None, (kind, str(t), o, g, bad)
            for g in untouched.tolist():
                assert hs.moment_check(kind, t, None, rows.values[g], rows.saw_null[g], **o) is None
            continue
        if kind in hs.LIST_KINDS:
            mine = hs.list_reference(kind, ids, vals, groups, **{k: v for k, v in o.items() if k == "mode"})
            got = mine.take(pa.array(present))
            if kind == "hash_distinct":  # the binary's order inside a distinct list is its hash table's
                assert [sorted(map(repr, x)) for x in got.to_pylist()] == [sorted(map(repr, x)) for x in want.to_pylist()]
            else:
                gr.assert_same_lists(got, want)
            assert all(len(x) == 0 for x in mine.take(pa.array(untouched)).to_pylist())
            continue
        mine = hs.reference(kind, ids, vals, groups, **o)
        if want.type != mine.type:
            want = want.cast(mine.type)
        hs.assert_result(kind, mine.take(pa.array(present)), want, msg=f"{kind} {t} {o}")
        ident = hs.identity(kind, o.get("skip_nulls", True), o.get("min_count", 1))
        tail = mine.take(pa.array(untouched))
        if ident is None:
            assert tail.null_count == len(tail)
        elif isinstance(ident, float):
            assert np.isnan(tail.to_numpy(zero_copy_only=False)).all() and tail.null_count == 0
        else:
            assert set(tail.to_pylist()) == {ident}


def test_plan_constants():
    assert hs.MIN_CAP & (hs.MIN_CAP - 1) == 0 and hs.MIN_CAP <= hs.K_PRIVATE_MAX_GROUPS
    assert hs.K_MOMENT_PRIVATE_GROUPS == hs.K_PRIVATE_MAX_GROUPS
    assert 0 < hs.PRIVATE_MIN_ROWS < hs.HASHAGG_BAND_MIN_ROWS == hs.MOMENT_BAND_MIN_ROWS
    assert hs.COUNT_BAND_BYTES_PER_GROUP < hs.BAND_BYTES_PER_GROUP and hs.MOMENT_STATE_PLANES == 5
    # millions of groups take more than one band for every kind, hash_count included
    assert hs.G_BIG > hs.HASHAGG_BAND_BYTES // hs.COUNT_BAND_BYTES_PER_GROUP and hs.G_BIG >= 1_000_000


def device_schedules():
    for kind, t in hs.MATRIX:
        yield kind, t, hs.options(kind), hs.schedule(kind, t, hs.seed_of(kind, t)), False
    for kind, t, o in hs.BANDED:
        yield kind, t, [o], hs.schedule(kind, t, hs.seed_of(kind, t, True), banded=True), True


def test_device_schedules_reach_every_path_and_growth():
    reached = {}
    for kind, t, opts_list, steps, banded in device_schedules():
        resizes = [s.groups for s in steps if s.op == "resize"]
        cap = hs.MIN_CAP
        assert resizes[0] < cap and resizes == sorted(resizes), (kind, t)
        for g in (cap, cap + 1, 2 * cap, 2 * cap + 1):
            assert g in resizes, (kind, t, g)
        assert resizes[-1] == resizes[-2] == steps[-1].groups >= 1_000_000 and steps[-1].op == "resize"
        layouts = {s.batch.layout for s in steps if s.op == "consume"}
        assert {"sliced", "valid_no_nulls", "all_null"} <= layouts and any(s.batch.n == 0 for s in steps if s.op == "consume")
        # some groups no batch touches, and a batch of old ids only right after the large growth
        ids, _ = hs.concat(steps)
        assert len(np.unique(ids)) < steps[-1].groups
        big = [i for i, s in enumerate(steps) if s.op == "resize" and s.groups == resizes[-1]][0]
        assert int(steps[big + 1].batch.ids.max()) < resizes[-3]
        for o in opts_list:
            plan = [p for s, p in hs.planned_paths(kind, t, steps, o.get("skip_nulls", True)) if s.op == "consume" and s.batch.n]
            fams = [hs.path_family(p.path) for p in plan]
            for f in fams:
                reached.setdefault(kind, set()).add(f)
            if len(hs.kind_paths(kind, t) - (set() if banded else {"banded"})) > 1:
                # a path adds into state another path wrote
                assert any(a != b for a, b in zip(fams, fams[1:])), (kind, t, fams)
    for kind, t, _, _, _ in device_schedules():
        assert hs.kind_paths(kind, t) <= reached[kind], (kind, hs.kind_paths(kind, t) - reached[kind])
    # every kind of the C ABI is streamed
    from arrow_b200 import _cabi
    assert set(_cabi.HASH_AGG_KINDS) == {k for k, _ in hs.MATRIX}
