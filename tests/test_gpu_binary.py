"""Parity of the var-binary (utf8 / binary, 32- and 64-bit offsets) and dictionary
selection kernels through the C-ABI, against the oracle and the reference binary."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from oracle import arrow_oracle as ora
from tests.util import SEED, assert_equal, random_array

pytestmark = pytest.mark.gpu
STRING_TYPES = [pa.string(), pa.large_string(), pa.binary(), pa.large_binary()]


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_binary_filter(ctx, t):
    v = pa.array(["a", "bb", None, "", "ccc"], pa.string()).cast(t)
    for m in ([0, 1, 0, 1, 1], [1, None, 1, 0, 1], [None] * 5, [0] * 5, [1] * 5):
        mask = pa.array([None if x is None else bool(x) for x in m], pa.bool_())
        for ns in ("drop", "emit_null"):
            got = bc.filter(dev(v, ctx), dev(mask, ctx), ns).to_arrow()
            assert_equal(got, pc.filter(v, mask, null_selection_behavior=ns), f"{m} {ns}")
    assert len(bc.filter(dev(v.slice(0, 0), ctx), dev(pa.array([], pa.bool_()), ctx)).to_arrow()) == 0
    for n, lo, hi in ((1500, 0, 32), (50000, 0, 32), (9000, 0, 3), (3000, 100, 400)):
        for null_p in (0.0, 0.1, 0.9):
            vals = random_array(t, n, null_p, SEED + n, lo=lo, hi=hi, offset=3)
            for true_p, mask_null in ((0.5, 0.0), (0.05, 0.05), (0.999, 0.3)):
                mask = random_array(pa.bool_(), n, mask_null, SEED + 1, hi=true_p, offset=2)
                for ns in ("drop", "emit_null"):
                    got = bc.filter(dev(vals, ctx), dev(mask, ctx), ns)
                    want = ora.filter(vals, mask, ns)
                    assert_equal(got.to_arrow(), want, f"{t} n={n} {null_p} {true_p} {ns}")
                    assert got.null_count == want.null_count
                    assert_equal(got.to_arrow(), pc.filter(vals, mask, null_selection_behavior=ns))


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_binary_take(ctx, t):
    v = pa.array(["a", "bb", None, "", "ccc"], pa.string()).cast(t)
    for idx in ([0, 1, 0], [4, None, 2, 3], [], [1] * 9):
        i = pa.array(idx, pa.int8())
        assert_equal(bc.take(dev(v, ctx), dev(i, ctx)).to_arrow(), pc.take(v, i), str(idx))
    with pytest.raises(pa.ArrowIndexError) as want:
        pc.take(v, pa.array([0, 5], pa.int32()))
    with pytest.raises(pa.ArrowIndexError) as got:
        bc.take(dev(v, ctx), dev(pa.array([0, 5], pa.int32()), ctx))
    assert str(got.value) == str(want.value)
    for n, n_idx in ((1025, 257), (30000, 70000)):
        for null_p in (0.0, 0.05, 0.95):
            vals = random_array(t, n, null_p, SEED, offset=1)
            for it in (pa.int16(), pa.uint32(), pa.int64()):
                hi = min(n - 1, np.iinfo(it.to_pandas_dtype()).max)
                idx = random_array(it, n_idx, null_p, SEED + 5, lo=0, hi=hi, offset=3)
                got = bc.take(dev(vals, ctx), dev(idx, ctx))
                want = ora.take(vals, idx)
                assert_equal(got.to_arrow(), want, f"{t} {it} {null_p}")
                assert got.null_count == want.null_count
                assert_equal(got.to_arrow(), pc.take(vals, idx))


def test_dictionary_filter_take(ctx):
    # BASELINE config 5's second half: dictionary-encoded Take moves the index column only
    dictionary = pa.array([f"value-{i}" for i in range(1000)])
    for it in (pa.int8(), pa.int32(), pa.int64()):
        hi = min(999, np.iinfo(it.to_pandas_dtype()).max)
        d = pa.DictionaryArray.from_arrays(random_array(it, 20000, 0.1, SEED, lo=0, hi=hi), dictionary)
        dd = dev(d, ctx)
        mask = random_array(pa.bool_(), 20000, 0.05, SEED + 1, hi=0.5)
        for ns in ("drop", "emit_null"):
            assert_equal(bc.filter(dd, dev(mask, ctx), ns).to_arrow(), pc.filter(d, mask, null_selection_behavior=ns))
        idx = random_array(pa.int64(), 5000, 0.1, SEED + 2, lo=0, hi=19999)
        assert_equal(bc.take(dd, dev(idx, ctx)).to_arrow(), pc.take(d, idx))
        assert_equal(bc.take(dd, dev(idx, ctx)).to_arrow(), ora.take(d, idx))


@pytest.mark.parametrize("shift", [1, 3, 5])
def test_binary_filter_unaligned_data_buffer(ctx, shift):
    """A byte buffer that does not start on an 8-byte boundary takes the byte-wise copy
    path instead of the aligned-word path; both must agree with the reference."""
    t = pa.large_string()
    n = 20000
    vals = random_array(t, n, 0.1, SEED + shift, lo=0, hi=40)
    mask = random_array(pa.bool_(), n, 0.05, SEED + 9, hi=0.5)
    aligned = dev(vals, ctx)
    data = np.frombuffer(vals.buffers()[2], dtype=np.uint8)
    raw = ctx.alloc(len(data) + 16)
    host = np.ascontiguousarray(data)
    ctx.h2d(raw.ptr + shift, host.ctypes.data, len(host))
    ctx.sync()
    moved = DeviceArray.from_pointers(ctx, t, n, aligned.buffers[1].ptr, validity_ptr=aligned.buffers[0].ptr,
                                      null_count=vals.null_count, data2_ptr=raw.ptr + shift, keepalive=(aligned, raw))
    for ns in ("drop", "emit_null"):
        want = pc.filter(vals, mask, null_selection_behavior=ns)
        assert_equal(bc.filter(moved, dev(mask, ctx), ns).to_arrow(), want, ns)
        assert_equal(bc.filter(aligned, dev(mask, ctx), ns).to_arrow(), want, ns)
    idx = random_array(pa.int32(), 5000, 0.05, SEED + 2, lo=0, hi=n - 1)
    assert_equal(bc.take(moved, dev(idx, ctx)).to_arrow(), pc.take(vals, idx))


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_binary_filter_take_long_rows_large_tiles(ctx, t):
    """the tile copy of Filter and Take on rows longer than 32 bytes, 100-400-byte rows and tiles whose output exceeds
    36 KB, with nulls, emit_null and null indices"""
    for n, lo, hi in ((1500, 0, 32), (50000, 0, 32), (9000, 0, 3), (3000, 100, 400), (20000, 0, 70)):
        for null_p in (0.0, 0.1):
            vals = random_array(t, n, null_p, SEED + n, lo=lo, hi=hi, offset=3)
            for true_p, mask_null in ((0.5, 0.0), (0.999, 0.3)):
                mask = random_array(pa.bool_(), n, mask_null, SEED + 1, hi=true_p, offset=2)
                for ns in ("drop", "emit_null"):
                    assert_equal(bc.filter(dev(vals, ctx), dev(mask, ctx), ns).to_arrow(), ora.filter(vals, mask, ns),
                                 f"{t} n={n} {lo}-{hi} {null_p} {true_p} {ns}")
            idx = random_array(pa.int64(), n // 2 + 7, null_p, SEED + 5, lo=0, hi=n - 1, offset=3)
            assert_equal(bc.take(dev(vals, ctx), dev(idx, ctx)).to_arrow(), ora.take(vals, idx), f"take {t} n={n}")


def test_large_binary_values_beyond_4gib_are_refused(ctx):
    """64-bit offsets: the selection kernels stage lengths / offsets tile-relative in 32 bits, so a tile whose value bytes
    reach 4 GiB must be reported, not wrapped (ADVICE r1).  The offsets below CLAIM a 5 GiB value; only the sizes pass
    runs before the error, so the (tiny) data buffer is never dereferenced."""
    import torch
    offs_t = torch.tensor([0, 3, 3 + (5 << 30), 8 + (5 << 30), 9 + (5 << 30)], dtype=torch.int64, device="cuda")
    data_t = torch.full((64,), ord("x"), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    d = DeviceArray.from_pointers(ctx, pa.large_binary(), 4, offs_t.data_ptr(), data2_ptr=data_t.data_ptr())
    with pytest.raises(pa.ArrowNotImplementedError, match="4 GiB"):
        bc.filter(d, DeviceArray.from_arrow(pa.array([True, True, False, True]), ctx))
    with pytest.raises(pa.ArrowNotImplementedError, match="4 GiB"):
        bc.take(d, DeviceArray.from_arrow(pa.array([0, 1], pa.int32()), ctx))
    # rows that do not touch the huge value are fine for take (its tiles are about the TAKEN rows)
    got = bc.take(d, DeviceArray.from_arrow(pa.array([0, 0], pa.int32()), ctx)).to_arrow()
    assert got.to_pylist() == [b"xxx", b"xxx"]
