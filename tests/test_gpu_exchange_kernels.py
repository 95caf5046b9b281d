"""Sender-side kernels of the multi-GPU exchange: b2_range_split (stable split of (value, row) pairs by range id) and
b2_hash_partition (owner rank of each group-by key)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from tests import exact_ref as er
from tests import sort_ref
from tests.hash_keys import fmix64_np
from tests.util import SEED, random_array

pytestmark = pytest.mark.gpu


def _hash_partition(ctx, arr, n_parts):
    from arrow_b200 import DeviceArray, _cabi as cabi
    from arrow_b200.device import check
    keys = DeviceArray.from_arrow(arr, ctx)     # holds the device buffers until the kernel has read them
    ca, out = keys._c(), cabi.B2Array()
    check(ctx.lib.b2_hash_partition(ctx.handle, C.byref(ca), n_parts, C.byref(out), ctx.stream))
    return DeviceArray._from_c(ctx, out, pa.uint32()).to_arrow()


# every width; negative signed keys must not be sign-extended, and float keys hash their bits (-0.0 and +0.0 apart)
@pytest.mark.parametrize("t", sort_ref.NUMERIC, ids=str)
@pytest.mark.parametrize("n_parts", [1, 3, 8, 1000])
@pytest.mark.parametrize("n,null_p,offset", [(0, 0.0, 0), (1, 0.0, 0), (100_003, 0.0, 0), (100_003, 0.1, 5), (4099, 0.5, 13)])
def test_hash_partition_hashes_the_zero_extended_bits(ctx, t, n_parts, n, null_p, offset):
    rng = np.random.default_rng(SEED + n + offset)
    arr = sort_ref.edge_array(t, n, rng, null_p=null_p, offset=offset)
    got = _hash_partition(ctx, arr, n_parts)
    assert got.type == pa.uint32() and len(got) == n and got.null_count == 0
    ids = (fmix64_np(er.bits(arr).astype(np.uint64)) % np.uint64(n_parts)).astype(np.uint32)
    want = np.where(er.valid_mask(arr), ids, 0)                    # null keys belong to partition 0
    bad = np.flatnonzero(got.to_numpy() != want)
    assert len(bad) == 0, f"{len(bad)} of {n} ids differ, first rows {bad[:5].tolist()}: bits " \
                          f"{[hex(int(x)) for x in er.bits(arr)[bad[:5]]]} got {got.to_numpy()[bad[:5]].tolist()} want {want[bad[:5]].tolist()}"


@pytest.mark.parametrize("n_parts", [0, -1])
def test_hash_partition_refuses_fewer_than_one_part(ctx, n_parts):
    with pytest.raises(pa.ArrowInvalid, match="n_parts"):
        _hash_partition(ctx, pa.array([1, 2, 3], pa.int64()), n_parts)


@pytest.mark.parametrize("t", [pa.int64(), pa.float64(), pa.int16(), pa.uint32()], ids=str)
@pytest.mark.parametrize("n,n_split,null_p,offset", [(0, 1, 0.0, 0), (1, 0, 0.0, 0), (2049, 1, 0.1, 3), (100_003, 3, 0.1, 1), (300_000, 7, 0.0, 0),
                                                     (50_000, 15, 0.5, 5)])
def test_range_split_is_a_stable_partition(ctx, t, n, n_split, null_p, offset):
    from arrow_b200 import DeviceArray, _cabi as cabi
    from arrow_b200.device import check
    from oracle import arrow_oracle as ora
    vals = random_array(t, n, null_p, SEED + n, lo=0, hi=1000, offset=offset)
    rng = np.random.default_rng(SEED)
    sp = np.sort(rng.integers(0, 1000, n_split)).astype(t.to_pandas_dtype())
    splitters = pa.array(sp, t)
    row_base = 12345
    dv, ds = DeviceArray.from_arrow(vals, ctx), DeviceArray.from_arrow(splitters, ctx)
    counts = (C.c_int64 * (n_split + 2))()
    cv, cs, ov, orows = dv._c(), ds._c(), cabi.B2Array(), cabi.B2Array()
    check(ctx.lib.b2_range_split(ctx.handle, C.byref(cv), C.byref(cs), 0, row_base, C.byref(ov), C.byref(orows), counts, ctx.stream))
    got_v = DeviceArray._from_c(ctx, ov, t).to_arrow()
    got_r = DeviceArray._from_c(ctx, orows, pa.uint32()).to_arrow().to_numpy().astype(np.int64)
    v, valid = ora.values(vals), ora.validity(vals)
    ids = np.where(valid, np.searchsorted(sp, v, side="right"), n_split + 1)
    order = np.argsort(ids, kind="stable")
    assert list(counts) == np.bincount(ids, minlength=n_split + 2).tolist()
    assert (got_r == order + row_base).all()
    n_valid = int(valid.sum())
    got_vals = got_v.to_numpy(zero_copy_only=False)
    if pa.types.is_floating(t):
        assert np.array_equal(got_vals[:n_valid], v[order][:n_valid], equal_nan=True)
    else:
        assert (got_vals[:n_valid] == v[order][:n_valid]).all()
