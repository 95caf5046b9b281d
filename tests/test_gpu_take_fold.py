"""The folded gather of b2_take_cast_arith (take_partitioned.cu pass F): a cast to float32 of float64 / int64 values with
nulls gathers from a float32 copy of the values in which each null row's slot is a signalling NaN naming the row's cast
in a side table.  Forced with B2_TAKE_PARTITION=1 and KB-sized bands, and compared bit for bit with the direct kernels
(B2_TAKE_PARTITION=0), every slot included: a null row's slot holds cast(values[j]) op other[i] on both paths."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi

from .util import SEED

pytestmark = pytest.mark.gpu

FOLD_LAUNCHES = 3  # count, scan, fold

SPECIAL_BITS = [
    0x7FF8000000000000, 0xFFF8000000000000,  # quiet NaN of both signs
    0x7FF8000000000123, 0xFFFC0000DEADBEEF,  # quiet NaN with payloads
    0x7FF0000000000001, 0xFFF0000000000001,  # signalling NaN of both signs
    0x7FF4000000000000, 0xFFF7FFFFFFFFFFFF,  # signalling NaN with high / full payloads
    0x7FF0000000000000, 0xFFF0000000000000,  # +-inf
    0x0000000000000000, 0x8000000000000000,  # +-0
    0x0000000000000001, 0x800FFFFFFFFFFFFF,  # double subnormals (cast to +-0)
]
SPECIAL_DOUBLES = [1e-40, -1e-45, 1.17549435e-38, 1e39, -1e300, 3.4028235677973366e38, -3.4028234663852886e38,
                   np.finfo(np.float64).max, 2.0 ** 24 + 1]


def _values(t, vlen, offset, rng, valid):
    """vlen values of t after `offset` leading rows; `valid` covers all offset + vlen rows (None: no bitmap)"""
    m = offset + vlen
    if t == pa.float64():
        data = rng.uniform(-1e6, 1e6, m)
        bits = data.view(np.uint64)
        k = np.arange(m) % 5 == 0  # every fifth row special, null or not
        pool = np.array(SPECIAL_BITS + [np.float64(d).view(np.uint64) for d in SPECIAL_DOUBLES], np.uint64)
        bits[k] = pool[rng.integers(0, len(pool), int(k.sum()))]
    else:
        data = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, m, dtype=np.int64, endpoint=True)
        data[::7] = rng.integers(-(1 << 24), 1 << 24, len(data[::7]))
    vbuf = None if valid is None else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    nulls = 0 if valid is None else int((~valid).sum())
    arr = pa.Array.from_buffers(t, m, [vbuf, pa.py_buffer(data.tobytes())], null_count=nulls)
    return arr.slice(offset) if offset else arr


def _call(monkeypatch, partition, band_kb, fn):
    monkeypatch.setenv("B2_TAKE_PARTITION", partition)
    if partition == "1":
        monkeypatch.setenv("B2_TAKE_PART_BAND_KB", str(band_kb))
    else:
        monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
    lib = _cabi.lib()
    before = lib.b2_launch_count()
    out = fn().to_arrow()
    return out, lib.b2_launch_count() - before


def _same_bits(a, b):
    """every slot's bits and every validity bit (Array.equals would call two NaN slots different)"""
    assert len(a) == len(b) and a.null_count == b.null_count
    assert a.buffers()[1].to_pybytes()[a.offset * 4:(a.offset + len(a)) * 4] == \
        b.buffers()[1].to_pybytes()[b.offset * 4:(b.offset + len(b)) * 4]
    if a.null_count:
        va = np.unpackbits(np.frombuffer(a.buffers()[0], np.uint8), bitorder="little")[a.offset:a.offset + len(a)]
        vb = np.unpackbits(np.frombuffer(b.buffers()[0], np.uint8), bitorder="little")[b.offset:b.offset + len(b)]
        assert np.array_equal(va, vb)


def _check(ctx, monkeypatch, values, idx, other, band_kb, folds=True):
    dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, other))
    for op in ("add", "subtract", "multiply"):
        fold, n_fold = _call(monkeypatch, "1", band_kb, lambda: bc.take_cast_arith(dv, di, pa.float32(), op, do))
        direct, _ = _call(monkeypatch, "0", band_kb, lambda: bc.take_cast_arith(dv, di, pa.float32(), op, do))
        _same_bits(fold, direct)
    # the same take cast to float64 never folds: the partitioned passes without pass F
    other64 = DeviceArray.from_arrow(other.cast(pa.float64()), ctx)
    _, n_plain = _call(monkeypatch, "1", band_kb, lambda: bc.take_cast_arith(dv, di, pa.float64(), "add", other64))
    assert n_fold - n_plain == (FOLD_LAUNCHES if folds else 0)


def _indices(rng, n, vlen, offset, null_p):
    raw = rng.integers(0, vlen, offset + n)
    mask = rng.random(offset + n) < null_p if null_p else None
    arr = pa.array(raw, pa.int64(), mask=mask)
    return arr.slice(offset) if offset else arr


def _other(rng, n):
    return pa.array(rng.uniform(-10, 10, n).astype(np.float32), pa.float32(), mask=rng.random(n) < 0.1)


# (value type, values_length, n, slice offset, index null p, band KB): 4 KB bands hold 1024 folded rows
CASES = [
    (pa.float64(), 70001, 200003, 0, 0.0, 4),
    (pa.float64(), 70001, 200003, 13, 0.1, 4),   # bitmap offset not 0
    (pa.float64(), 5000, 4097, 3, 0.05, 1),      # 256-row bands, tiles smaller than 4096
    (pa.float64(), 9999, 30000, 0, 0.0, 64),     # one band
    (pa.int64(), 70001, 200003, 5, 0.1, 4),
    (pa.int64(), 12289, 50000, 0, 0.0, 16),      # 4096-row bands: one count tile per band
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_fold_equals_direct(ctx, monkeypatch, case):
    t, vlen, n, off, inull, band_kb = CASES[case]
    rng = np.random.default_rng(SEED + case)
    band_rows = (band_kb << 10) // 4
    valid = rng.random(off + vlen) >= 0.1
    if vlen > 8 * band_rows:
        valid[off + 2 * band_rows:off + 3 * band_rows] = False  # a band entirely null
        valid[off + 5 * band_rows:off + 6 * band_rows] = True   # a band with no nulls
    _check(ctx, monkeypatch, _values(t, vlen, off, rng, valid), _indices(rng, n, vlen, off, inull), _other(rng, n),
           band_kb)


def test_fold_without_nulls_or_known_null_count(ctx, monkeypatch):
    """no nulls, or a null count the slice does not know: the partitioned path without pass F"""
    rng = np.random.default_rng(SEED)
    vlen, n = 20000, 40000
    idx, other = _indices(rng, n, vlen, 0, 0.1), _other(rng, n)
    _check(ctx, monkeypatch, _values(pa.float64(), vlen, 0, rng, None), idx, other, 4, folds=False)
    valid = rng.random(vlen + 7) >= 0.1
    dv = DeviceArray.from_arrow(_values(pa.float64(), vlen + 7, 0, rng, valid), ctx).slice(7)
    assert dv.null_count == -1
    di, do = DeviceArray.from_arrow(idx, ctx), DeviceArray.from_arrow(other, ctx)
    part, _ = _call(monkeypatch, "1", 4, lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do))
    direct, _ = _call(monkeypatch, "0", 4, lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do))
    _same_bits(part, direct)


def test_fold_full_sentinel_range(ctx, monkeypatch):
    """a 2^22-row band entirely null: its last row's rank, 2^22 - 1, takes the first negative sentinel"""
    rng = np.random.default_rng(SEED + 99)
    vlen, n = (1 << 22) + 3000, 1 << 20
    valid = np.zeros(vlen, bool)
    valid[(1 << 22) + rng.integers(0, 3000, 50)] = True
    raw = rng.integers(0, vlen, n)
    raw[:4096] = np.arange((1 << 22) - 4096, 1 << 22)  # the band's last rows: its highest ranks
    _check(ctx, monkeypatch, _values(pa.float64(), vlen, 0, rng, valid), pa.array(raw, pa.int64()), _other(rng, n),
           16 << 10)


def test_device_cast_makes_no_sentinel(ctx):
    """float64 -> float32 on the device quiets every NaN, so no valid row's cast reads as a sentinel"""
    bits = np.array(SPECIAL_BITS, np.uint64)
    arr = pa.Array.from_buffers(pa.float64(), len(bits), [None, pa.py_buffer(bits.tobytes())])
    got = bc.cast(DeviceArray.from_arrow(arr, ctx), pa.float32(), safe=False).to_arrow()
    f = np.frombuffer(got.buffers()[1], np.uint32)[got.offset:got.offset + len(bits)]
    assert not (((f & 0x7FC00000) == 0x7F800000) & ((f & 0x3FFFFF) != 0)).any()
    assert ((f & 0x7FC00000) == 0x7FC00000).sum() == 8  # the eight NaNs, quiet


def test_fold_index_error(ctx, monkeypatch):
    rng = np.random.default_rng(SEED)
    vlen, n = 50_000, 30_000
    valid = rng.random(vlen) >= 0.1
    values = _values(pa.float64(), vlen, 0, rng, valid)
    raw = rng.integers(0, vlen, n)
    raw[7777], raw[20001] = vlen + 5, vlen  # the first out-of-range valid index is named
    mask = np.zeros(n, bool)
    mask[100] = True
    raw[100] = vlen + 99                    # a null index is never checked
    idx = pa.array(raw, pa.int64(), mask=mask)
    with pytest.raises(pa.ArrowIndexError) as want:
        pc.take(values, idx)
    dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, _other(rng, n)))
    msgs = []
    for partition in ("1", "0"):
        with pytest.raises(pa.ArrowIndexError) as err:
            _call(monkeypatch, partition, 4, lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do))
        msgs.append(str(err.value))
    assert msgs[0] == msgs[1] == str(want.value)
