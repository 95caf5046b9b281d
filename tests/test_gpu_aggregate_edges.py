"""Hash aggregates, the fused group-by, the Grouper, unique / value_counts / dictionary_encode, the hash join and b2_reduce
at the edges where kernels go wrong, against EXACT references (tests/exact_ref.py): NaN of several payloads, +-inf, -0.0 /
+0.0 and denormals as values and as keys, float sums whose exact value does not depend on the order of the additions, and
integers over their whole range (sums wrap mod 2^64).  Results compare bit-exactly; any NaN equals any NaN, and for
min / max -0.0 equals +0.0.

The hash aggregates are driven through each consume regime of hash_aggregate.cu launch_consume: the shared-memory private
copy (<= 2048 groups, >= 2^14 rows), plain atomics (more groups, < 2^24 rows), L2 bands of group ids (>= 2^24 rows and
more than 24 MB / 16 B = 1.57M groups), the dense packed path of integer hash_sum (>= 2^22 rows, 8- and 16-bit values),
and merge of two partial states."""
from fractions import Fraction
from functools import lru_cache

import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from oracle import arrow_oracle as ora
from tests import exact_ref as er
from tests.test_aggregate_edges_oracle import acero_by_id, kat_cases, sorted_by_key, special_keys
from tests.util import INT_TYPES, SEED

pytestmark = pytest.mark.gpu
FLOATS = [pa.float32(), pa.float64()]
FNS = ("hash_sum", "hash_mean", "hash_min", "hash_max", "hash_product", "hash_count", "hash_count_distinct")
OPTS = [(True, 1), (True, 0), (True, 3), (False, 1), (False, 0), (False, 3)]
# (groups, rows) per consume regime; "banded" must stay above 24 MB / 16 B groups and 2^24 rows
REGIMES = {"private": (2000, 1 << 16), "atomic": (20_000, 300_000), "banded": (1_600_000, (1 << 24) + 5)}


def dev(a, ctx):
    return DeviceArray.from_arrow(a, ctx)


def agg_opts(fn, skip_nulls, min_count):
    if fn in ("hash_count", "hash_count_distinct"):
        return {"mode": "only_valid"}
    return {"skip_nulls": skip_nulls, "min_count": min_count}


def device_agg(ctx, fn, vals, ids, groups, opts):
    agg = bc.HashAggregator(fn, vals.type, ctx=ctx, **opts)
    agg.resize(groups)
    agg.consume(dev(vals, ctx), dev(pa.array(ids, pa.uint32()), ctx))
    return agg.finalize().to_arrow()


def device_merged(ctx, fn, vals, ids, groups, opts):
    """two partial states -- the first half of the rows, and the second half with its group ids reversed -- merged through
    a mapping that undoes the reversal"""
    h = len(ids) // 2 + 1
    a = bc.HashAggregator(fn, vals.type, ctx=ctx, **opts)
    a.resize(groups)
    a.consume(dev(vals.slice(0, h), ctx), dev(pa.array(ids[:h], pa.uint32()), ctx))
    b = bc.HashAggregator(fn, vals.type, ctx=ctx, **opts)
    b.resize(groups)
    b.consume(dev(vals.slice(h), ctx), dev(pa.array((groups - 1 - ids[h:].astype(np.int64)).astype(np.uint32)), ctx))
    a.merge(b, dev(pa.array((groups - 1 - np.arange(groups)).astype(np.uint32)), ctx))
    return a.finalize().to_arrow()


def reference_agg(fn, vals, ids, groups, opts):
    if fn == "hash_count_distinct":
        return pa.array(er.count_distinct(ids, vals, groups, opts["mode"]))
    return ora.hash_aggregate(fn, vals, pa.array(ids, pa.uint32()), groups, **opts)


@lru_cache(maxsize=2)
def special_data(vt_name, groups, n):
    return er.special_float_groups(np.dtype(vt_name), groups, n, SEED + groups)


# ---- A. float values with NaN / +-inf / +-0 / denormals through every consume regime --------------------------------------
def check_special(ctx, vt, groups, n, opt_list, merged=False, acero=True):
    ids, vals = special_data(vt.to_pandas_dtype().__name__, groups, n)
    all_nan = np.arange(groups) % len(er.GROUP_CLASSES) == er.GROUP_CLASSES.index("all_nan")
    for skip_nulls, min_count in opt_list:
        for fn in FNS:
            if fn == "hash_count_distinct" and n > (1 << 20):
                continue   # its state is a Grouper over (value, group) pairs, not the regimes under test here
            if fn in ("hash_count", "hash_count_distinct") and (skip_nulls, min_count) != opt_list[0]:
                continue   # no options besides the count mode
            opts = agg_opts(fn, skip_nulls, min_count)
            got = (device_merged if merged else device_agg)(ctx, fn, vals, ids, groups, opts)
            msg = f"{fn} {vt} n={n} groups={groups} {opts}{' merged' if merged else ''}"
            mm = fn in ("hash_min", "hash_max")
            er.assert_same(got, reference_agg(fn, vals, ids, groups, opts), zeros_equal=mm, msg=msg + " vs oracle")
            if acero:
                er.assert_same(got, acero_by_id(ids, vals, fn, opts), zeros_equal=mm, msg=msg + " vs acero")
            if mm:   # a group whose values are all NaN is NaN, never +-inf
                r = er.raw(got)[all_nan & er.valid_mask(got)]
                assert len(r) and np.isnan(r).all(), msg + ": NaN-only groups"


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("regime", ["private", "atomic"])
def test_special_float_values(ctx, vt, regime):
    groups, n = REGIMES[regime]
    check_special(ctx, vt, groups, n, OPTS)


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_special_float_values_merge(ctx, vt):
    check_special(ctx, vt, 20_000, 300_000, [(True, 1), (False, 3), (True, 0)], merged=True)


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_special_float_values_l2_bands(ctx, vt):
    groups, n = REGIMES["banded"]
    check_special(ctx, vt, groups, n, [(True, 0), (False, 3)], acero=False)


@pytest.mark.parametrize("case", kat_cases(), ids=lambda c: c[0])
def test_kat_minmax_nan_device(ctx, case):
    """the reference's GroupBy.MinOrMax / MinMaxWithNaN vectors through the Grouper path and through the private regime
    (the same rows repeated 2^12 times: at least 2^14 rows)"""
    _, keys, vals, ek, emin, emax = case
    for reps in (1, 1 << 12):
        k_in = pa.concat_arrays([keys] * reps)
        v_in = pa.concat_arrays([vals] * reps)
        (uk,), (mn, mx) = bc.group_by([dev(k_in, ctx)], [("hash_min", dev(v_in, ctx), None), ("hash_max", dev(v_in, ctx), None)],
                                      fused=False)
        k, mn, mx = sorted_by_key(uk.to_arrow(), mn.to_arrow(), mx.to_arrow())
        er.assert_same(k, ek, msg="keys")
        er.assert_same(mn, emin, msg=f"hash_min x{reps}")
        er.assert_same(mx, emax, msg=f"hash_max x{reps}")


# ---- B. float sums whose exact value is order independent -----------------------------------------------------------------
def int_valued(rng, n, dtype, bound=1 << 20):
    return rng.integers(-bound, bound + 1, n).astype(dtype)


def exact_float_sums(ids, v, valid, groups):
    """integer-valued floats: the exact sum as an int64 (|partial sums| < 2^53), then as a double"""
    s = np.zeros(groups, np.int64)
    np.add.at(s, ids[valid], v[valid].astype(np.int64))
    return s.astype(np.float64)


def keys_to_ids(keys: pa.Array):
    """group ids by key BITS, null key last: (ids, number of groups, a key array indexed by id)"""
    ok = er.valid_mask(keys)
    ub, inv = np.unique(er.bits(keys), return_inverse=True)
    ids = np.where(ok, inv, len(ub)).astype(np.int64)
    present = np.unique(ids)
    remap = np.full(len(ub) + 1, -1)
    remap[present] = np.arange(len(present))
    ids = remap[ids]
    first = np.zeros(len(present), np.int64)
    first[ids[::-1]] = np.arange(len(ids))[::-1]
    return ids, len(present), keys.take(pa.array(first))


def check_keyed_sums(got_keys, got_sum, got_count, keys, v, valid, msg=""):
    ids, groups, ukeys = keys_to_ids(keys)
    want_sum = exact_float_sums(ids, v, valid, groups)
    cnt = np.bincount(ids[valid], minlength=groups)
    go, wo = pa.array(er.key_order(got_keys)), pa.array(er.key_order(ukeys))
    er.assert_same(got_keys.take(go), ukeys.take(wo), msg=msg + " keys")
    er.assert_same(got_count.take(go), pa.array(cnt).take(wo), msg=msg + " counts")
    er.assert_same(got_sum.take(go), pa.array(want_sum, mask=cnt == 0).take(wo), msg=msg + " sums")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("groups", [7, 600, 300_000])
def test_float_sums_exact_fused(ctx, vt, groups):
    """GroupBySumCount over float values (general / atomic paths): per-group sums far past 2^24 are exact in double"""
    n = 3_000_000
    rng = np.random.default_rng(SEED + groups)
    keys = pa.array(rng.integers(0, groups, n, dtype=np.int64), mask=rng.random(n) < 0.01)
    v = int_valued(rng, n, vt.to_pandas_dtype())
    valid = rng.random(n) >= 0.1
    g = bc.GroupBySumCount(pa.int64(), vt, expected_groups=groups, ctx=ctx)
    g.consume(dev(keys, ctx), dev(pa.array(v, mask=~valid), ctx))
    paths = g.path_counts()
    assert paths["dense"] == 0 and paths["compact"] == 0 and sum(paths.values()) == 1, paths
    k, s, c = [x.to_arrow() for x in g.finalize()]
    check_keyed_sums(k, s, c, keys, v, valid, msg=f"fused {vt} {groups}")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("groups", [1000, 50_000])
def test_float_sums_exact_grouper(ctx, vt, groups):
    """Grouper + hash_sum / hash_mean (private regime at 1000 groups, atomics at 50 000)"""
    n = 1 << 21
    rng = np.random.default_rng(SEED + 3 * groups)
    keys = pa.array(rng.integers(-groups, groups, n, dtype=np.int64) // 2)
    v = int_valued(rng, n, vt.to_pandas_dtype())
    valid = rng.random(n) >= 0.1
    vals = dev(pa.array(v, mask=~valid), ctx)
    (uk,), (s, m, c) = bc.group_by([dev(keys, ctx)], [("hash_sum", vals, None), ("hash_mean", vals, None), ("hash_count", vals, None)],
                                   fused=False)
    uk, s, m, c = uk.to_arrow(), s.to_arrow(), m.to_arrow(), c.to_arrow()
    check_keyed_sums(uk, s, c, keys, v, valid, msg=f"grouper {vt} {groups}")
    # mean = exact sum / count, rounded once
    ids, ng, ukeys = keys_to_ids(keys)
    cnt = np.bincount(ids[valid], minlength=ng)
    with np.errstate(all="ignore"):
        want_m = exact_float_sums(ids, v, valid, ng) / cnt
    go, wo = pa.array(er.key_order(uk)), pa.array(er.key_order(ukeys))
    er.assert_same(m.take(go), pa.array(want_m, mask=cnt == 0).take(wo), msg="hash_mean")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("n,offset", [((1 << 24) + 3, 0), ((1 << 24) + 3, 1), (1_000_003, 3)])
def test_float_reduce_exact(ctx, vt, n, offset):
    """b2_reduce sum / mean: exact at 2^24 + 3 values and at unaligned offsets (a float32 accumulator would round)"""
    rng = np.random.default_rng(SEED + n + offset)
    v = int_valued(rng, n + offset, vt.to_pandas_dtype())
    mask = rng.random(n + offset) < 0.05
    arr = pa.array(v, mask=mask)
    d = dev(arr, ctx).slice(offset)
    vv = v[offset:][~mask[offset:]]
    exact = int(vv.astype(np.int64).sum())
    assert bc.sum(d).as_py() == float(exact)
    assert bc.mean(d).as_py() == np.float64(exact) / np.float64(len(vv))
    assert bc.min_max(d).as_py() == {"min": float(vv.min()), "max": float(vv.max())}


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_float_sums_cancellation_bound(ctx, vt):
    """x, -x and small residues: |got - fsum| <= (c - 1) 2^-53 sum|x| per group of c values (the bound any order of c - 1
    double additions meets); pyarrow's row-order sums must meet it too"""
    import pyarrow.acero  # noqa: F401
    rng = np.random.default_rng(SEED + 77)
    groups, n_x = 8000, 400_000
    x = (rng.standard_normal(n_x) * 10.0 ** rng.integers(-3, 12, n_x)).astype(vt.to_pandas_dtype())
    resid = (rng.standard_normal(n_x // 4) * 1e-3).astype(x.dtype)
    v = np.concatenate([x, -x, resid])
    ids = rng.integers(0, groups, n_x)
    ids = np.concatenate([ids, rng.permutation(ids), rng.integers(0, groups, n_x // 4)]).astype(np.uint32)
    perm = rng.permutation(len(v))
    v, ids = v[perm], ids[perm]
    vals = pa.array(v)
    want = np.array(er.fsums(ids, v, groups))
    absum = np.zeros(groups)
    np.add.at(absum, ids, np.abs(v.astype(np.float64)))
    cnt = np.bincount(ids, minlength=groups)
    bound = (cnt - 1) * 2.0 ** -53 * absum
    g = bc.GroupBySumCount(pa.int64(), vt, ctx=ctx)
    g.consume(dev(pa.array(ids.astype(np.int64)), ctx), dev(vals, ctx))
    k, s, _ = [x.to_arrow() for x in g.finalize()]
    fused = np.zeros(groups)
    fused[k.to_numpy()] = s.to_numpy()
    outs = {"atomic hash_sum": device_agg(ctx, "hash_sum", vals, ids, groups, {}), "fused": pa.array(fused),
            "acero": acero_by_id(ids, vals, "hash_sum", {})}
    for name, got in outs.items():
        err = np.abs(er.raw(got).astype(np.float64) - want)
        assert (err <= bound).all(), (name, int(np.argmax(err - bound)), float((err - bound).max()))
    # the private regime needs <= 2048 groups: the same rows folded into 1500 groups, with their own bound
    ids2 = (ids % 1500).astype(np.uint32)
    want2 = np.array(er.fsums(ids2, v, 1500))
    absum2 = np.zeros(1500)
    np.add.at(absum2, ids2, np.abs(v.astype(np.float64)))
    bound2 = (np.bincount(ids2, minlength=1500) - 1) * 2.0 ** -53 * absum2
    err2 = np.abs(er.raw(device_agg(ctx, "hash_sum", vals, ids2, 1500, {})) - want2)
    assert (err2 <= bound2).all(), ("private", float((err2 - bound2).max()))


# ---- C. integers over their whole range, bit-exact ------------------------------------------------------------------------
def full_range(rng, t, n, null_probability=0.1):
    """values over the type's whole range, salted with its min and max; sums wrap mod 2^64 in int64 / uint64"""
    dt = np.dtype(t.to_pandas_dtype())
    info = np.iinfo(dt)
    v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
    salt = rng.random(n)
    v[salt < 0.02] = info.min
    v[(salt >= 0.02) & (salt < 0.04)] = info.max
    return v, rng.random(n) >= null_probability


def want_int_sums(ids, v, valid, groups):
    signed = np.issubdtype(v.dtype, np.signedinteger)
    sums = er.exact_int_sums(ids[valid], v[valid], groups)
    cnt = np.bincount(ids[valid], minlength=groups)
    acc = np.array([er.wrap64(s, signed) for s in sums], dtype=np.int64 if signed else np.uint64)
    return pa.array(acc, mask=cnt == 0), cnt


FUSED_PATHS = {  # (default, B2_GROUPBY_DENSE=0, both off) for 150 000 groups over 4.5M rows
    1: ("dense", "compact", "general"), 2: ("dense", "compact", "general"),
    4: ("compact", "compact", "general"),    # 32-bit values: the packed dense word has no room for 2^22-row sub-batches
    8: ("general", "general", "general"),    # full-range 64-bit values fit no window: the sampled value range is 2^64
}


@pytest.mark.parametrize("t", INT_TYPES, ids=str)
def test_full_range_ints_fused_paths(ctx, t, monkeypatch):
    n, groups = 4_500_000, 150_000
    rng = np.random.default_rng(SEED + t.bit_width + pa.types.is_signed_integer(t))
    keys = pa.array(rng.integers(0, groups, n, dtype=np.int64), mask=rng.random(n) < 0.01)
    v, valid = full_range(rng, t, n)
    vals = pa.array(v, mask=~valid)
    ids, ng, ukeys = keys_to_ids(keys)
    want, cnt = want_int_sums(ids, v, valid, ng)
    wo = pa.array(er.key_order(ukeys))
    for env, want_path in zip(({}, {"B2_GROUPBY_DENSE": "0"}, {"B2_GROUPBY_DENSE": "0", "B2_GROUPBY_COMPACT": "0"}),
                              FUSED_PATHS[t.bit_width // 8]):
        for k in ("B2_GROUPBY_DENSE", "B2_GROUPBY_COMPACT"):
            monkeypatch.delenv(k, raising=False)
        for k, x in env.items():
            monkeypatch.setenv(k, x)
        g = bc.GroupBySumCount(pa.int64(), t, expected_groups=groups, ctx=ctx)
        g.consume(dev(keys, ctx), dev(vals, ctx))
        paths = g.path_counts()
        assert paths[want_path] == 1 and sum(paths.values()) == 1, (env, paths)
        k, s, c = [x.to_arrow() for x in g.finalize()]
        go = pa.array(er.key_order(k))
        er.assert_same(k.take(go), ukeys.take(wo), msg=f"{t} {env} keys")
        er.assert_same(c.take(go), pa.array(cnt).take(wo), msg=f"{t} {env} counts")
        er.assert_same(s.take(go), want.take(wo), msg=f"{t} {env} sums")


def test_path_settings_are_per_group_by(ctx, monkeypatch):
    """B2_GROUPBY_DENSE is read when a group-by is created: one created with it set stays off the dense path after another
    is created without it"""
    n, groups = 4_500_000, 150_000
    rng = np.random.default_rng(SEED + 150)
    keys = pa.array(rng.integers(0, groups, n, dtype=np.int64), mask=rng.random(n) < 0.01)
    v = rng.integers(-100, 101, n).astype(np.int64)
    valid = rng.random(n) >= 0.1
    ids, ng, ukeys = keys_to_ids(keys)
    want, cnt = want_int_sums(ids, v, valid, ng)
    wo = pa.array(er.key_order(ukeys))
    monkeypatch.setenv("B2_GROUPBY_DENSE", "0")
    a = bc.GroupBySumCount(pa.int64(), pa.int64(), expected_groups=groups, ctx=ctx)
    monkeypatch.delenv("B2_GROUPBY_DENSE")
    b = bc.GroupBySumCount(pa.int64(), pa.int64(), expected_groups=groups, ctx=ctx)
    dk, dv = dev(keys, ctx), dev(pa.array(v, mask=~valid), ctx)
    for name, g, dense in (("A", a, 0), ("B", b, 1)):
        g.consume(dk, dv)
        paths = g.path_counts()
        assert paths["dense"] == dense and sum(paths.values()) == 1, (name, paths)
        k, s, c = [x.to_arrow() for x in g.finalize()]
        go = pa.array(er.key_order(k))
        er.assert_same(k.take(go), ukeys.take(wo), msg=f"{name} keys")
        er.assert_same(c.take(go), pa.array(cnt).take(wo), msg=f"{name} counts")
        er.assert_same(s.take(go), want.take(wo), msg=f"{name} sums")


INT_REGIMES = {  # (groups, rows) of Grouper + hash_sum
    "dense_by_id": (100_000, (1 << 22) + 17),    # 8- and 16-bit values take the packed dense path, wider ones the atomics
    "private": (1000, 1 << 20),
    "atomic": (50_000, 1 << 21),
    "banded": REGIMES["banded"],
}


@pytest.mark.parametrize("t", INT_TYPES, ids=str)
@pytest.mark.parametrize("regime", list(INT_REGIMES) + ["merge"])
def test_full_range_ints_hash_sum(ctx, t, regime, monkeypatch):
    groups, n = INT_REGIMES.get(regime, (50_000, 1 << 21))
    if regime == "banded":
        monkeypatch.setenv("B2_GROUPBY_DENSE", "0")   # else 8- and 16-bit values take the dense path at this size
    rng = np.random.default_rng(SEED + groups + t.bit_width)
    ids = rng.integers(0, groups, n).astype(np.uint32)
    v, valid = full_range(rng, t, n)
    vals = pa.array(v, mask=~valid)
    want, _ = want_int_sums(ids, v, valid, groups)
    got = (device_merged if regime == "merge" else device_agg)(ctx, "hash_sum", vals, ids, groups, {})
    er.assert_same(got, want, msg=f"hash_sum {t} {regime}")


@pytest.mark.parametrize("t", INT_TYPES, ids=str)
def test_full_range_ints_reduce(ctx, t):
    n, offset = (1 << 20) + 3, 1
    rng = np.random.default_rng(SEED + 5 + t.bit_width)
    v, valid = full_range(rng, t, n + offset)
    d = dev(pa.array(v, mask=~valid), ctx).slice(offset)
    vv = v[offset:][valid[offset:]]
    signed = pa.types.is_signed_integer(t)
    assert bc.sum(d).as_py() == er.wrap64(sum(int(x) for x in vv.tolist()), signed)
    assert bc.min_max(d).as_py() == {"min": int(vv.min()), "max": int(vv.max())}


def test_full_range_int64_mean(ctx):
    """hash_mean accumulates in double (GroupedMeanAccType): within (c + 1) 2^-53 sum|x| / c of the exact mean"""
    groups, n = 1000, 1 << 20
    rng = np.random.default_rng(SEED + 64)
    ids = rng.integers(0, groups, n).astype(np.uint32)
    v, valid = full_range(rng, pa.int64(), n)
    got = er.raw(device_agg(ctx, "hash_mean", pa.array(v, mask=~valid), ids, groups, {}))
    sums = er.exact_int_sums(ids[valid], v[valid], groups)
    cnt = np.bincount(ids[valid], minlength=groups)
    absum = np.zeros(groups)
    np.add.at(absum, ids[valid], np.abs(v[valid].astype(np.float64)))
    for g in range(groups):
        err = abs(Fraction(float(got[g])) - Fraction(sums[g], int(cnt[g])))
        assert err <= Fraction((cnt[g] + 1) * absum[g] / cnt[g]) * Fraction(1, 2 ** 53), (g, float(err))


# ---- D. float keys group by bytes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_float_keys_grouper(ctx, vt):
    """consume / lookup / get_uniques: 0.0 and -0.0, and NaNs of different payloads, are different groups; the all-ones
    pattern (the 8-byte table's empty marker) is an ordinary key"""
    keys = special_keys(vt, 300_000, SEED + 91)
    gr = bc.Grouper([vt], ctx=ctx)
    ids = gr.consume([dev(keys, ctx)]).to_arrow()
    (uniq,) = [u.to_arrow() for u in gr.get_uniques()]
    ok = er.valid_mask(keys)
    assert gr.num_groups == len(np.unique(er.bits(keys)[ok])) + 1
    back = uniq.take(ids)
    assert np.array_equal(er.valid_mask(back), ok)
    assert np.array_equal(er.bits(back)[ok], er.bits(keys)[ok])
    look = gr.lookup([dev(keys.slice(1000, 5000), ctx)]).to_arrow()
    assert look.equals(ids.slice(1000, 5000))
    unseen = pa.array(np.array([3.25, -7.5], vt.to_pandas_dtype()))
    assert gr.lookup([dev(unseen, ctx)]).to_arrow().null_count == 2
    # and hash_sum over those ids equals the oracle's per key
    vals = pa.array(np.arange(len(keys), dtype=np.int64))
    (uk,), (s,) = bc.group_by([dev(keys, ctx)], [("hash_sum", dev(vals, ctx), None)], fused=False)
    (ok_,), (os_,) = ora.group_by([keys], [("hash_sum", vals, None)])
    go, wo = pa.array(er.key_order(uk.to_arrow())), pa.array(er.key_order(ok_))
    er.assert_same(uk.to_arrow().take(go), ok_.take(wo), msg="uniques")
    er.assert_same(s.to_arrow().take(go), os_.take(wo), msg="sums")


@pytest.mark.parametrize("name,vt,base,span,special,n,want_path", [
    ("f32-denormal-band", pa.float32(), 0x00000000, 200_000, False, 4_500_000, "dense"),   # +0.0 and the denormals
    ("f64-narrow-band", pa.float64(), 0x3FF0000000000000, 200_000, False, 3_000_000, "compact"),
    ("f64-specials", pa.float64(), 0x3FF0000000000000, 200_000, True, 3_000_000, "general"),
])
def test_float_keys_fused(ctx, name, vt, base, span, special, n, want_path):
    """GroupBySumCount with float keys: the dense path samples key BITS and does not look at the key type"""
    rng = np.random.default_rng(SEED + span + n)
    ut = er.UINT_OF_WIDTH[vt.bit_width // 8]
    kb = (np.uint64(base) + rng.integers(0, span, n).astype(np.uint64)).astype(ut)
    if special:
        kb[rng.integers(0, n, 20_000)] = rng.choice(er.bits(er.special_values(vt.to_pandas_dtype())), 20_000)
    keys = pa.array(kb.view(vt.to_pandas_dtype()), mask=rng.random(n) < 0.01)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    valid = rng.random(n) >= 0.1
    g = bc.GroupBySumCount(vt, pa.int64(), expected_groups=span, ctx=ctx)
    g.consume(dev(keys, ctx), dev(pa.array(v, mask=~valid), ctx))
    paths = g.path_counts()
    assert paths[want_path] == 1 and sum(paths.values()) == 1, paths
    k, s, c = [x.to_arrow() for x in g.finalize()]
    ids, ng, ukeys = keys_to_ids(keys)
    want, cnt = want_int_sums(ids, v, valid, ng)
    go, wo = pa.array(er.key_order(k)), pa.array(er.key_order(ukeys))
    er.assert_same(k.take(go), ukeys.take(wo), msg=name + " keys")
    er.assert_same(c.take(go), pa.array(cnt).take(wo), msg=name + " counts")
    er.assert_same(s.take(go), want.take(wo), msg=name + " sums")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
def test_float_keys_vector_hash(ctx, vt):
    arr = special_keys(vt, 100_000, SEED + 93)
    d = dev(arr, ctx)
    er.assert_same(bc.unique(d).to_arrow(), ora.unique(arr), msg="unique")
    values, counts = bc.value_counts(d)
    want = ora.value_counts(arr)
    er.assert_same(values.to_arrow(), want.field("values"), msg="value_counts.values")
    er.assert_same(counts.to_arrow(), want.field("counts"), msg="value_counts.counts")
    for enc in ("mask", "encode"):
        got = bc.dictionary_encode(d, enc).to_arrow()
        w = ora.dictionary_encode(arr, enc)
        er.assert_same(got.indices, w.indices, msg=f"dictionary_encode.indices {enc}")
        er.assert_same(got.dictionary, w.dictionary, msg=f"dictionary_encode.dictionary {enc}")


@pytest.mark.parametrize("vt", FLOATS, ids=str)
@pytest.mark.parametrize("join_type", ["inner", "left outer", "left semi", "left anti", "full outer"])
def test_float_keys_hash_join(ctx, vt, join_type):
    """-0.0 does not match 0.0; a NaN matches an identical NaN only"""
    from tests.test_gpu_hash_join import check
    check(ctx, [special_keys(vt, 3000, SEED + 95)], [special_keys(vt, 500, SEED + 96)], join_type)
