"""Hash join with a residual filter and null-equal keys on the device (b2_hash_join_ex + b2_join_residual, csrc/hash_join.cu):
exact equality with the row reference (tests/join_ref.py: order, null slots and null counts) and sorted equality with the
reference binary's hashjoin node with filter_expression."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import join_ref
from tests.test_join_residual_oracle import ACERO_TYPES, SWAPPED, acero_pairs, make_sides, rows_key

pytestmark = pytest.mark.gpu
JOIN_TYPES = ["inner", "left outer", "left semi", "left anti", "full outer"]


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


def assert_same(got, want, what):
    gl, gr = got
    wl, wr = want
    assert gl.to_arrow().equals(wl), what
    assert gl.null_count == wl.null_count, what
    if wr is None:
        assert gr is None, what
    else:
        assert gr.to_arrow().equals(wr), what
        assert gr.null_count == wr.null_count, what


def device_pairs(ctx, left_keys, right_keys, join_type, key_cmp=None, residual=None):
    """hash_join_indices on the device for the eight acero join types (RIGHT_* by swapping the sides), as the pairs
    ref_pairs gives"""
    dl, dr = [dev(k, ctx) for k in left_keys], [dev(k, ctx) for k in right_keys]
    if join_type in SWAPPED:
        swapped = None if residual is None else (lambda r, l: residual(l, r))
        a, b = bc.hash_join_indices(dr, dl, SWAPPED[join_type], key_cmp, swapped)
        a = a.to_arrow().to_pylist()
        return [(None, x) for x in a] if b is None else [(y, x) for x, y in zip(a, b.to_arrow().to_pylist())]
    a, b = bc.hash_join_indices(dl, dr, join_type, key_cmp, residual)
    a = a.to_arrow().to_pylist()
    return [(x, None) for x in a] if b is None else list(zip(a, b.to_arrow().to_pylist()))


def less_payload(ctx, lv: pa.Array, rv: pa.Array):
    """(device residual, host residual) for lv[l] < rv[r] -- null where either payload is null"""
    dlv, drv = dev(lv, ctx), dev(rv, ctx)
    hl, hr = lv.to_pylist(), rv.to_pylist()
    return (lambda l, r: bc.less(bc.take(dlv, l), bc.take(drv, r)),
            lambda l, r: None if hl[l] is None or hr[r] is None else hl[l] < hr[r])


def all_pass():
    return lambda l, r: bc.is_valid(l), lambda l, r: True


def none_pass():
    return lambda l, r: bc.is_null(l), lambda l, r: False


def check(ctx, left_keys, right_keys, join_types=JOIN_TYPES, key_cmp=None, residuals=()):
    for jt in join_types:
        for d_res, h_res in residuals:
            got = bc.hash_join_indices([dev(k, ctx) for k in left_keys], [dev(k, ctx) for k in right_keys], jt, key_cmp, d_res)
            assert_same(got, join_ref.hash_join_indices(left_keys, right_keys, jt, key_cmp, h_res), (jt, key_cmp))


@pytest.mark.parametrize("key_kind", ["int64", "utf8", "two"])
@pytest.mark.parametrize("join_type", ACERO_TYPES)
def test_matches_reference_binary(ctx, key_kind, join_type):
    """all eight join types against the stock hashjoin node with the same filter (sorted pairs) and the row reference"""
    left, right, lk, rk = make_sides(key_kind, seed=len(join_type) * 31 + len(key_kind), nl=3000, nr=2000)
    lkeys, rkeys = [left[c].combine_chunks() for c in lk], [right[c].combine_chunks() for c in rk]
    dres, hres = less_payload(ctx, left["lv"].combine_chunks(), right["rv"].combine_chunks())
    got = device_pairs(ctx, lkeys, rkeys, join_type, residual=dres)
    want = acero_pairs(left, right, lk, rk, join_type, pc.field("lv") < pc.field("rv"))
    assert rows_key(got) == rows_key(want), join_type
    if join_type not in SWAPPED:
        assert_same(bc.hash_join_indices([dev(k, ctx) for k in lkeys], [dev(k, ctx) for k in rkeys], join_type, None, dres),
                    join_ref.hash_join_indices(lkeys, rkeys, join_type, None, hres), join_type)


def test_empty_sides_and_no_candidates(ctx):
    rng = np.random.default_rng(1)
    k = pa.array(rng.integers(0, 50, 500), pa.int64())
    v = pa.array(rng.normal(size=500), pa.float64(), mask=rng.random(500) < 0.2)
    empty_k, empty_v = pa.array([], pa.int64()), pa.array([], pa.float64())
    check(ctx, [k], [empty_k], residuals=[less_payload(ctx, v, empty_v)])
    check(ctx, [empty_k], [k], residuals=[less_payload(ctx, empty_v, v)])
    check(ctx, [empty_k], [empty_k], residuals=[less_payload(ctx, empty_v, empty_v)])
    disjoint = pa.array(rng.integers(100, 150, 400), pa.int64())   # no key matches: no candidate pairs
    check(ctx, [k], [disjoint], residuals=[less_payload(ctx, v, v[:400]), all_pass()])


def test_all_pass_none_pass_and_null_results(ctx):
    rng = np.random.default_rng(2)
    lk = pa.array(rng.integers(0, 40, 3000), pa.int64(), mask=rng.random(3000) < 0.1)
    rk = pa.array(rng.integers(0, 60, 2500), pa.int64(), mask=rng.random(2500) < 0.1)
    lv = pa.array(rng.normal(size=3000), pa.float64(), mask=rng.random(3000) < 0.3)
    rv = pa.array(rng.normal(size=2500), pa.float64(), mask=rng.random(2500) < 0.3)
    check(ctx, [lk], [rk], residuals=[all_pass(), none_pass(), less_payload(ctx, lv, rv)])
    # all pass = the filter-free join
    for jt in JOIN_TYPES:
        assert_same(bc.hash_join_indices([dev(lk, ctx)], [dev(rk, ctx)], jt, None, all_pass()[0]),
                    tuple(x.to_arrow() if x is not None else None for x in bc.hash_join_indices([dev(lk, ctx)], [dev(rk, ctx)], jt)), jt)


def test_one_probe_row_with_100k_candidates(ctx):
    n = 100_003
    rng = np.random.default_rng(3)
    lk = pa.array([7, 3, 7], pa.int64())
    rk = pa.array(np.where(rng.random(n) < 0.98, 7, 5), pa.int64())
    lv = pa.array([0.0, 1.0, None], pa.float64())
    rv = pa.array(rng.normal(size=n), pa.float64(), mask=rng.random(n) < 0.1)
    check(ctx, [lk], [rk], residuals=[less_payload(ctx, lv, rv)])


@pytest.mark.parametrize("n_cand", [1, 31, 32, 33, 63, 64, 65, 4095, 4096, 4097, 8191, 12289])
def test_word_and_tile_edges(ctx, n_cand):
    """one candidate per left row, so the candidate count, the left side and the survivors cross 32-pair words and
    4096-row scan tiles"""
    rng = np.random.default_rng(n_cand)
    lk = pa.array(np.arange(n_cand), pa.int64())
    rk = pa.array(rng.permutation(n_cand + 5), pa.int64())
    lv = pa.array(rng.normal(size=n_cand), pa.float64(), mask=rng.random(n_cand) < 0.1)
    rv = pa.array(rng.normal(size=n_cand + 5), pa.float64())
    check(ctx, [lk], [rk], residuals=[less_payload(ctx, lv, rv), all_pass()])
    # every left row passing except the last one of each 32-pair word
    keep_host = lambda l, r: (l % 32) != 31  # noqa: E731
    dl = dev(pa.array(np.arange(n_cand) % 32, pa.int64()), ctx)
    keep_dev = lambda l, r: bc.not_equal(bc.take(dl, l), 31)  # noqa: E731
    check(ctx, [lk], [rk], residuals=[(keep_dev, keep_host)])


def test_null_equal_keys(ctx):
    rng = np.random.default_rng(4)
    n, m = 2000, 1500
    lk = pa.array(rng.integers(0, 30, n), pa.int64(), mask=rng.random(n) < 0.15)
    rk = pa.array(rng.integers(0, 30, m), pa.int64(), mask=rng.random(m) < 0.15)
    ls = pa.array([f"w{v}" for v in rng.integers(0, 5, n)], pa.utf8(), mask=rng.random(n) < 0.2)
    rs = pa.array([f"w{v}" for v in rng.integers(0, 5, m)], pa.utf8(), mask=rng.random(m) < 0.2)
    lv = pa.array(rng.normal(size=n), pa.float64(), mask=rng.random(n) < 0.2)
    rv = pa.array(rng.normal(size=m), pa.float64(), mask=rng.random(m) < 0.2)
    res = [(None, None), less_payload(ctx, lv, rv)]
    check(ctx, [lk], [rk], key_cmp=["is"], residuals=res)
    check(ctx, [ls], [rs], key_cmp=["is"], residuals=res)
    check(ctx, [lk, ls], [rk, rs], key_cmp=["is", "eq"], residuals=res)
    check(ctx, [lk, ls], [rk, rs], key_cmp=["eq", "is"], residuals=res)
    check(ctx, [lk, ls], [rk, rs], key_cmp=["is", "is"], residuals=res)
    # all EQ through key_cmp is the plain join
    for jt in JOIN_TYPES:
        assert_same(bc.hash_join_indices([dev(lk, ctx)], [dev(rk, ctx)], jt, ["eq"]),
                    join_ref.hash_join_indices([lk], [rk], jt), jt)


def test_invalid_candidates_are_refused(ctx):
    u32 = lambda xs: dev(pa.array(xs, pa.uint32()), ctx)  # noqa: E731
    keep = lambda n: dev(pa.array([True] * n), ctx)  # noqa: E731
    for jt in JOIN_TYPES:
        with pytest.raises(pa.ArrowInvalid, match="n_left"):
            bc.join_residual(u32([0, 1, 5]), u32([0, 0, 0]), keep(3), 5, 4, jt)
        with pytest.raises(pa.ArrowInvalid, match="n_right"):
            bc.join_residual(u32([0, 1, 2]), u32([0, 4, 0]), keep(3), 5, 4, jt)
        with pytest.raises(pa.ArrowInvalid, match="non-decreasing"):
            bc.join_residual(u32(list(range(40)) + [3] + list(range(41, 70))), u32([0] * 70), keep(70), 80, 4, jt)
        with pytest.raises(pa.ArrowInvalid, match="keep flags"):
            bc.join_residual(u32([0, 1, 2]), u32([0, 1]), keep(2), 5, 4, jt)
        with pytest.raises(pa.ArrowInvalid, match="keep flags"):
            bc.join_residual(u32([0, 1, 2]), u32([0, 1, 2]), keep(4), 5, 4, jt)
    # the context still works afterwards
    a, b = bc.join_residual(u32([0, 0, 2]), u32([1, 3, 0]), dev(pa.array([True, None, False]), ctx), 3, 4, "full outer")
    assert a.to_arrow().to_pylist() == [0, 1, 2, None, None, None]
    assert b.to_arrow().to_pylist() == [1, None, None, 0, 2, 3]
