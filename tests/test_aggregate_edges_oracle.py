"""CPU: the oracle's hash aggregates, scalar aggregates, unique / value_counts / dictionary_encode, Grouper and hash join
against the reference binary (pyarrow / Acero) on NaN (several payloads), +-inf, -0.0 / +0.0 and denormals, as values and
as keys -- the data the GPU tests in test_gpu_aggregate_edges.py compare the kernels with the oracle on.  Plus the
known-answer vectors of the reference's GroupBy.MinOrMax and GroupBy.MinMaxWithNaN tests."""
import json
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from oracle import arrow_oracle as ora
from tests import exact_ref as er
from tests.util import HERE, SEED

FLOATS = [pa.float32(), pa.float64()]
PA_NAME = {"hash_sum": "sum", "hash_mean": "mean", "hash_min": "min", "hash_max": "max", "hash_product": "product",
           "hash_count": "count", "hash_count_distinct": "count_distinct"}


def acero_by_id(ids, vals, fn, opts):
    """Acero's grouped `fn` keyed by the group ids, as an array indexed by group id (every group has rows)"""
    import pyarrow.acero  # noqa: F401
    if fn in ("hash_count", "hash_count_distinct"):
        o = pc.CountOptions(opts.get("mode", "only_valid"))
    else:
        o = pc.ScalarAggregateOptions(skip_nulls=opts.get("skip_nulls", True), min_count=opts.get("min_count", 1))
    t = pa.table({"g": pa.array(ids, pa.uint32()), "v": vals}).group_by("g", use_threads=False).aggregate([("v", PA_NAME[fn], o)])
    t = t.sort_by("g")
    assert t["g"].to_numpy().tolist() == list(range(len(t)))
    return t[f"v_{PA_NAME[fn]}"].combine_chunks()


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("skip_nulls,min_count", [(True, 1), (True, 0), (False, 1), (True, 3), (False, 3)])
def test_oracle_hash_aggregates_special_floats_vs_acero(vt, skip_nulls, min_count):
    groups = 60
    ids, vals = er.special_float_groups(vt.to_pandas_dtype(), groups, 1500, SEED + 1)
    opts = {"skip_nulls": skip_nulls, "min_count": min_count}
    for fn in ("hash_sum", "hash_mean", "hash_min", "hash_max", "hash_product"):
        want = acero_by_id(ids, vals, fn, opts)
        got = ora.hash_aggregate(fn, vals, pa.array(ids), groups, **opts)
        er.assert_same(got, want, zeros_equal=fn in ("hash_min", "hash_max"), msg=f"{fn} {vt} {opts}")
    for mode in ("only_valid", "only_null", "all"):
        want = acero_by_id(ids, vals, "hash_count_distinct", {"mode": mode})
        er.assert_same(ora.hash_aggregate("hash_count_distinct", vals, pa.array(ids), groups, mode=mode), want, msg=mode)
        er.assert_same(pa.array(er.count_distinct(ids, vals, groups, mode)), want, msg=f"exact_ref {mode}")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_oracle_all_nan_group_min_max_is_nan(vt):
    """the defect the ±inf start value hid: a group of NaNs only is NaN, not +inf / -inf"""
    vals = pa.array(np.array([np.nan, np.nan, 1.0, np.nan, -np.inf], dtype=vt.to_pandas_dtype()))
    ids = pa.array([0, 0, 1, 1, 2], pa.uint32())
    for fn, want in (("hash_min", [np.nan, 1.0, -np.inf]), ("hash_max", [np.nan, 1.0, -np.inf])):
        got = ora.hash_aggregate(fn, vals, ids, 3).to_pylist()
        assert np.isnan(got[0]) and got[1:] == want[1:], (fn, got)


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_oracle_scalar_aggregates_special_floats_vs_pyarrow(vt):
    dt = vt.to_pandas_dtype()
    rng = np.random.default_rng(SEED + 2)
    sv = er.special_values(dt)
    cases = {
        "all_nan": sv[2:6], "nan_and_finite": np.concatenate([sv[2:4], np.array([1.5, -2.0], dt)]),
        "infs": np.array([np.inf, -np.inf], dt), "pos_inf": np.array([np.inf, 1.0], dt), "neg_zero": np.array([-0.0, -0.0], dt),
        "zeros_neg_first": np.array([-0.0, 0.0], dt), "zeros_pos_first": np.array([0.0, -0.0], dt), "denormal": sv[-1:].repeat(5),
        "mixed": rng.permutation(np.concatenate([sv, rng.choice(np.array([0.5, -4.0, 2.0], dt), 20)])),
    }
    for name, v in cases.items():
        for mask in (None, np.arange(len(v)) % 3 == 1):
            arr = pa.array(v, mask=mask)
            for skip_nulls, min_count in ((True, 1), (False, 1), (True, 0), (True, 50)):
                o = pc.ScalarAggregateOptions(skip_nulls=skip_nulls, min_count=min_count)
                for fn, ofn in (("sum", ora.scalar_sum), ("mean", ora.scalar_mean)):
                    want = getattr(pc, fn)(arr, options=o)
                    got = ofn(arr, skip_nulls=skip_nulls, min_count=min_count)
                    er.assert_same(pa.array([got]), pa.array([want]), msg=f"{fn} {name} {mask is None} {skip_nulls} {min_count}")
                want = pc.min_max(arr, options=o)
                got = ora.scalar_min_max(arr, skip_nulls=skip_nulls, min_count=min_count)
                if name == "mixed" and want["min"].is_valid:
                    # "mixed" holds a signalling NaN: std::fmin / fmax make it a quiet NaN that replaces the running
                    # min / max, so the reference's result depends on where it sits (min 5e-324 with 0.0 present):
                    # check the documented rule, NaNs ignored, instead
                    vv = v[er.valid_mask(arr)]
                    want = {"min": pa.scalar(np.nanmin(vv), vt), "max": pa.scalar(np.nanmax(vv), vt)}
                for f in ("min", "max"):
                    er.assert_same(pa.array([got[f].as_py()], vt), pa.array([want[f].as_py()], vt), zeros_equal=True,
                                   msg=f"min_max.{f} {name}")


def special_keys(vt, n, seed, null_probability=0.05):
    """keys drawn from the special bit patterns and a few ordinary values"""
    dt = vt.to_pandas_dtype()
    rng = np.random.default_rng(seed)
    pool = np.concatenate([er.special_values(dt), np.array([1.0, -1.0, 2.5], dt)])
    return pa.array(rng.choice(pool, n), mask=rng.random(n) < null_probability)


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_oracle_vector_hash_float_keys_vs_pyarrow(vt):
    """0.0 / -0.0 and NaNs of different payloads are distinct values; first-occurrence order"""
    arr = special_keys(vt, 400, SEED + 3)
    er.assert_same(ora.unique(arr), pc.unique(arr), msg="unique")
    want_vc = pc.value_counts(arr)
    got_vc = ora.value_counts(arr)
    er.assert_same(got_vc.field("values"), want_vc.field("values"), msg="value_counts.values")
    er.assert_same(got_vc.field("counts"), want_vc.field("counts"), msg="value_counts.counts")
    for enc in ("mask", "encode"):
        want = pc.dictionary_encode(arr, null_encoding=enc)
        got = ora.dictionary_encode(arr, enc)
        er.assert_same(got.indices, want.indices, msg=f"dictionary_encode.indices {enc}")
        er.assert_same(got.dictionary, want.dictionary, msg=f"dictionary_encode.dictionary {enc}")
    n_bits = len(np.unique(er.bits(arr)[er.valid_mask(arr)]))
    assert len(pc.unique(arr)) == n_bits + 1   # + the null


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_oracle_grouper_and_join_float_keys_vs_acero(vt):
    import pyarrow.acero  # noqa: F401
    keys = special_keys(vt, 600, SEED + 4)
    vals = pa.array(np.arange(600, dtype=np.int64))
    gr = ora.Grouper([vt])
    ids = gr.consume([keys])
    (uniq,) = gr.get_uniques()
    # Take(uniques, ids) reproduces the keys bit for bit
    back = uniq.take(ids)
    assert np.array_equal(er.valid_mask(back), er.valid_mask(keys))
    assert np.array_equal(er.bits(back)[er.valid_mask(keys)], er.bits(keys)[er.valid_mask(keys)])
    # the same groups as Acero's: compare (key bits, sum) sorted by key bits
    want = pa.table({"k": keys, "v": vals}).group_by("k", use_threads=False).aggregate([("v", "sum")])
    osum = ora.hash_aggregate("hash_sum", vals, ids, gr.num_groups)
    wo, go = er.key_order(want["k"].combine_chunks()), er.key_order(uniq)
    er.assert_same(uniq.take(pa.array(go)), want["k"].combine_chunks().take(pa.array(wo)), msg="group keys")
    er.assert_same(osum.take(pa.array(go)), want["v_sum"].combine_chunks().take(pa.array(wo)), msg="group sums")
    # a join: -0.0 does not match 0.0, a NaN matches an identical NaN only
    right = special_keys(vt, 300, SEED + 5)
    lt = pa.table({"k": keys, "lrow": pa.array(np.arange(len(keys)))})
    rt = pa.table({"k": right, "rrow": pa.array(np.arange(len(right)))})
    ref = lt.join(rt, keys="k", join_type="inner", use_threads=False)
    want_pairs = sorted(zip(ref["lrow"].to_pylist(), ref["rrow"].to_pylist()))
    li, ri = ora.hash_join_indices([keys], [right], "inner")
    assert sorted(zip(li.to_pylist(), ri.to_pylist())) == want_pairs
    lb, rb = er.bits(keys), er.bits(right)
    assert all(lb[l] == rb[r] for l, r in want_pairs)


def kat_minmax():
    with open(os.path.join(HERE, "golden", "kat_minmax_nan.json")) as f:
        return json.load(f)


def kat_value(x):
    return {"NaN": float("nan"), "Inf": float("inf"), "-Inf": float("-inf")}.get(x, x) if isinstance(x, str) else x


def kat_cases():
    """(name, value type, keys, values, expected keys, expected min, expected max) of kat_minmax_nan.json"""
    d = kat_minmax()
    out = []
    for name in ("min_or_max", "min_max_with_nan"):
        c = d[name]
        for t in c.get("types", [c.get("type")]):
            vt = pa.float32() if t == "float" else pa.float64()
            keys = pa.array([r[1] for r in c["rows"]], pa.int64())
            vals = pa.array([kat_value(r[0]) for r in c["rows"]], vt)
            ek = pa.array([e[0] for e in c["expected"]], pa.int64())
            emin = pa.array([kat_value(e[1]) for e in c["expected"]], vt)
            emax = pa.array([kat_value(e[2]) for e in c["expected"]], vt)
            out.append((f"{name}-{t}", keys, vals, ek, emin, emax))
    return out


def sorted_by_key(keys, *cols):
    """rows sorted by key value, the null key last (the KAT's order)"""
    order = pa.array(np.lexsort((np.nan_to_num(keys.to_numpy(zero_copy_only=False).astype(np.float64), nan=0),
                                 ~er.valid_mask(keys))))
    return [keys.take(order)] + [c.take(order) for c in cols]


@pytest.mark.parametrize("case", kat_cases(), ids=lambda c: c[0])
def test_kat_minmax_nan_oracle(case):
    _, keys, vals, ek, emin, emax = case
    (uk,), (mn, mx) = ora.group_by([keys], [("hash_min", vals, None), ("hash_max", vals, None)])
    k, mn, mx = sorted_by_key(uk, mn, mx)
    er.assert_same(k, ek, msg="keys")
    er.assert_same(mn, emin, msg="hash_min")
    er.assert_same(mx, emax, msg="hash_max")
    # and the reference binary agrees with the vectors
    t = pa.table({"k": keys, "v": vals}).group_by("k", use_threads=False).aggregate([("v", "min"), ("v", "max")])
    k, mn, mx = sorted_by_key(t["k"].combine_chunks(), t["v_min"].combine_chunks(), t["v_max"].combine_chunks())
    er.assert_same(mn, emin, msg="acero hash_min")
    er.assert_same(mx, emax, msg="acero hash_max")
