"""CPU: the exact sort references of tests/sort_ref.py against the reference binary (pyarrow) and the oracle, on full-range
values with NaNs of both signs and several payloads, +-0, +-inf, subnormals and integer extremes, for every numeric type,
both orders and both null placements -- the references the GPU tests in test_gpu_sort_edges.py hold the kernels to."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from oracle import arrow_oracle as ora
from tests import sort_ref as sr
from tests import string_sort_oracle as sso
from tests.util import SEED

LENGTHS = (0, 1, 2, 500, 3001)


def _arr_list(x) -> list:
    return np.asarray(x.to_numpy(zero_copy_only=False), np.int64).tolist()


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_sort_indices_ref_matches_pyarrow_and_oracle(t):
    rng = np.random.default_rng(SEED + sr.NUMERIC.index(t))
    for n in LENGTHS:
        arr = sr.edge_array(t, n, rng, null_p=0.1, offset=n % 7)
        for order in sr.ORDERS:
            for placement in sr.PLACEMENTS:
                msg = f"{t} n={n} {order} {placement}"
                want = sr.sort_indices_ref(arr, order, placement)
                assert _arr_list(pc.array_sort_indices(arr, order=order, null_placement=placement)) == want, msg
                assert _arr_list(ora.sort_indices(arr, order, placement)) == want, msg
                assert sr.sort_indices_np(arr, order, placement).tolist() == want, msg


@pytest.mark.parametrize("placement", sr.PLACEMENTS)
def test_multi_key_ref_matches_pyarrow_and_oracle(placement):
    rng = np.random.default_rng(SEED + 100)
    for n in LENGTHS:
        cols = sr.multi_columns(n, rng)
        for keys in sr.MULTI_KEYS:
            msg = f"n={n} {keys} {placement}"
            names = [k for k, _ in keys]
            want = sr.sort_indices_multi_ref([cols[k] for k in names], [o for _, o in keys], placement)
            got = pc.sort_indices(pa.table({k: cols[k] for k in names}), sort_keys=keys, null_placement=placement)
            assert _arr_list(got) == want, msg
            assert _arr_list(sso.sort_indices_multi(cols, keys, placement)) == want, msg
            if "s" not in names:
                assert _arr_list(ora.sort_indices_multi(cols, keys, placement)) == want, msg
                assert sr.sort_indices_multi_np([cols[k] for k in names], [o for _, o in keys], placement).tolist() == want, msg


def test_multi_key_ties_fall_through_nan_payloads_and_signed_zeros():
    nan_a, nan_b = (np.array([b], np.uint64).view(np.float64)[0] for b in (0x7FF8000000000000, 0xFFF800000000BEEF))
    f = pa.array(np.array([nan_a, 0.0, nan_b, -0.0, nan_a, 0.0], np.float64))
    i = pa.array([5, 4, 3, 2, 1, 0], pa.int64())
    for placement in sr.PLACEMENTS:
        want = sr.sort_indices_multi_ref([f, i], ["ascending", "ascending"], placement)
        zeros, nans = [5, 3, 1], [4, 2, 0]                 # ordered by the second key
        assert want == (zeros + nans if placement == "at_end" else nans + zeros)
        assert _arr_list(pc.sort_indices(pa.table({"f": f, "i": i}), sort_keys=[("f", "ascending"), ("i", "ascending")],
                                         null_placement=placement)) == want


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_select_k_ref_matches_pyarrow_and_oracle(t):
    rng = np.random.default_rng(SEED + 200 + sr.NUMERIC.index(t))
    for n in LENGTHS:
        arr = sr.edge_array(t, n, rng, null_p=0.1, offset=3)
        vals, valid = sr.column(arr)
        plain = sum(sr.value_class(v, ok) == sr.VALUE for v, ok in zip(vals, valid.tolist()))
        for order in sr.ORDERS:
            for placement in sr.PLACEMENTS:
                for k in (0, 1, 10, n // 3, n + 4):
                    want = sr.select_k_ref(arr, k, order, placement)
                    assert _arr_list(ora.select_k_unstable(arr, k, order, placement)) == want, (t, n, order, placement, k)
            for k in (1, 10, n // 3):
                if k == 0 or k > plain:
                    continue
                # the reference's selection is unstable: compare the selected values (their sort keys) only
                got = _arr_list(pc.select_k_unstable(arr, k, [("x", order)]))
                keys = [sr.sort_key(vals[i], True, order, "at_end") for i in got]
                want = [sr.sort_key(vals[i], True, order, "at_end") for i in sr.select_k_ref(arr, k, order)]
                assert sorted(keys) == want, (t, n, order, k)


def _splitter_cases(t, rng):
    pool = sr.edge_pool(t)
    yield []
    yield [pool[len(pool) // 2]]
    yield list(pool[rng.integers(0, len(pool), 30)])                     # duplicates, and (floats) +-0, NaNs, +-inf
    yield list(np.sort(pool[rng.integers(0, len(pool), 63)]))


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_range_bin_ref_is_monotone_along_the_sort(t):
    rng = np.random.default_rng(SEED + 300 + sr.NUMERIC.index(t))
    arr = sr.edge_array(t, 4000, rng, null_p=0.1, offset=5, edge_p=0.6)
    vals, _ = sr.column(arr)
    for order in sr.ORDERS:
        perm = sr.sort_indices_ref(arr, order, "at_end")
        for sp in _splitter_cases(t, rng):
            sp = [v.item() for v in sp]
            bins = sr.range_bin_ref(arr, sp, order)
            along = [bins[i] for i in perm]
            assert along == sorted(along), (t, order, sp)
            assert set(bins) <= set(range(len(sp) + 2))
            assert sr.range_bins_np(arr, sp, order).tolist() == bins, (t, order, sp)
            if pa.types.is_floating(t):   # a NaN row passes every splitter, NaN splitters included
                assert all(b == len(sp) for b, v, ok in zip(bins, vals, sr.column(arr)[1]) if ok and v != v)


def test_range_bin_ref_known_answers():
    vals = pa.array([0.0, -0.0, float("nan"), -float("inf"), float("inf"), None, 1.0], pa.float64())
    sp = [-0.0, 0.0, float("nan"), float("inf")]
    assert sr.range_bin_ref(vals, sp, "ascending") == [2, 2, 4, 0, 3, 5, 2]
    assert sr.range_bin_ref(vals, sp, "descending") == [3, 3, 4, 3, 1, 5, 1]
    ints = pa.array([-(1 << 63), 0, (1 << 63) - 1], pa.int64())
    assert sr.range_bin_ref(ints, [-(1 << 63), (1 << 63) - 1], "ascending") == [1, 1, 2]
    assert sr.range_bin_ref(ints, [-(1 << 63), (1 << 63) - 1], "descending") == [2, 1, 1]


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_vectorised_forms_match_the_sorted_forms(t):
    rng = np.random.default_rng(SEED + 400 + sr.NUMERIC.index(t))
    arr = sr.edge_array(t, 30000, rng, null_p=0.2, offset=6)
    other = sr.edge_array(pa.int16(), 30000, rng, null_p=0.1, offset=1, edge_p=0.9)
    for order in sr.ORDERS:
        for placement in sr.PLACEMENTS:
            assert sr.sort_indices_np(arr, order, placement).tolist() == sr.sort_indices_ref(arr, order, placement)
            orders = [order, sr.ORDERS[1 - sr.ORDERS.index(order)]]
            assert (sr.sort_indices_multi_np([arr, other], orders, placement).tolist() ==
                    sr.sort_indices_multi_ref([arr, other], orders, placement))
