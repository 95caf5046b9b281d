"""The partitioned path of b2_take / b2_take_cast_arith (take_partitioned.cu), forced with B2_TAKE_PARTITION=1 and a
KB-sized band (B2_TAKE_PART_BAND_KB) so small inputs span many buckets: results, null counts and the IndexError must be
bit-identical to the direct kernels (B2_TAKE_PARTITION=0) and equal to the reference."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from oracle import arrow_oracle as ora

from .util import SEED, random_array

pytestmark = pytest.mark.gpu

# (values_length, n, values null p, index null p, other null p, slice offset, band KB)
CASES = [
    (1000, 1, 0.1, 0.0, 0.1, 0, 1),
    (1000, 300, 0.1, 0.1, 0.1, 0, 64),          # one bucket
    (5000, 4095, 0.1, 0.05, 0.1, 3, 1),
    (5000, 4096, 0.0, 0.05, 0.0, 0, 2),
    (5000, 4097, 0.1, 0.05, 0.1, 5, 1),
    (70001, 200003, 0.1, 0.1, 0.1, 1, 4),        # values_length not a multiple of the band
    (70000, 131072, 0.3, 0.0, 0.0, 0, 1),        # capped at 256 buckets: the band grows
]


def _run(monkeypatch, partition, band_kb, fn):
    monkeypatch.setenv("B2_TAKE_PARTITION", partition)
    if partition == "1":
        monkeypatch.setenv("B2_TAKE_PART_BAND_KB", str(band_kb))
    else:
        monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
    return fn().to_arrow()


def _same_bits(a, b):
    assert a.equals(b) and a.null_count == b.null_count
    width = a.type.bit_width // 8
    da, db = a.buffers()[1], b.buffers()[1]
    off_a, off_b = a.offset * width, b.offset * width
    assert da.to_pybytes()[off_a:off_a + len(a) * width] == db.to_pybytes()[off_b:off_b + len(b) * width]


@pytest.mark.parametrize("vt", [pa.float64(), pa.float32(), pa.int64(), pa.int32()], ids=str)
@pytest.mark.parametrize("it", [pa.int32(), pa.uint32(), pa.int64(), pa.uint64()], ids=str)
@pytest.mark.parametrize("to", [pa.float32(), pa.float64()], ids=str)
def test_fused_partitioned_equals_direct(ctx, monkeypatch, vt, it, to):
    for n_v, n, vnull, inull, onull, off, band_kb in CASES:
        values = random_array(vt, n_v, vnull, SEED + n, lo=-1000, hi=1000, offset=off)
        idx = random_array(it, n, inull, SEED + 1, lo=0, hi=n_v - 1, offset=off)
        other = random_array(to, n, onull, SEED + 2, lo=-10, hi=10, offset=2 * off)
        dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, other))
        for op in ("add", "subtract", "multiply"):
            part = _run(monkeypatch, "1", band_kb, lambda: bc.take_cast_arith(dv, di, to, op, do))
            direct = _run(monkeypatch, "0", band_kb, lambda: bc.take_cast_arith(dv, di, to, op, do))
            _same_bits(part, direct)
            want = pc.call_function(op, [pc.cast(pc.take(values, idx), to, safe=False), other])
            assert part.equals(want), f"{vt} {it} {to} {op} n={n}"
            assert part.null_count == want.null_count


@pytest.mark.parametrize("vt", [pa.float64(), pa.float32(), pa.int64(), pa.int32()], ids=str)
@pytest.mark.parametrize("it", [pa.int32(), pa.uint32(), pa.int64(), pa.uint64()], ids=str)
def test_take_partitioned_equals_direct(ctx, monkeypatch, vt, it):
    for n_v, n, vnull, inull, _, off, band_kb in CASES:
        values = random_array(vt, n_v, vnull, SEED + n, lo=-1000, hi=1000, offset=off)
        idx = random_array(it, n, inull, SEED + 1, lo=0, hi=n_v - 1, offset=off)
        dv, di = DeviceArray.from_arrow(values, ctx), DeviceArray.from_arrow(idx, ctx)
        part = _run(monkeypatch, "1", band_kb, lambda: bc.take(dv, di))
        direct = _run(monkeypatch, "0", band_kb, lambda: bc.take(dv, di))
        _same_bits(part, direct)
        want = ora.take(values, idx)
        assert part.equals(want), f"{vt} {it} n={n}"
        assert part.null_count == want.null_count


def test_scalar_other_partitioned(ctx, monkeypatch):
    values = random_array(pa.float64(), 9000, 0.1, SEED, lo=-1000, hi=1000)
    idx = random_array(pa.int64(), 20000, 0.1, SEED + 1, lo=0, hi=8999)
    dv, di = DeviceArray.from_arrow(values, ctx), DeviceArray.from_arrow(idx, ctx)
    other = pa.scalar(2.5, pa.float32())
    part = _run(monkeypatch, "1", 1, lambda: bc.take_cast_arith(dv, di, pa.float32(), "multiply", other))
    direct = _run(monkeypatch, "0", 1, lambda: bc.take_cast_arith(dv, di, pa.float32(), "multiply", other))
    _same_bits(part, direct)


@pytest.mark.parametrize("it", [pa.int32(), pa.int64(), pa.uint64()], ids=str)
def test_index_error_partitioned(ctx, monkeypatch, it):
    rng = np.random.default_rng(SEED)
    n_v, n = 50_000, 30_000
    values = pa.array(rng.uniform(0, 1e6, n_v), mask=rng.random(n_v) < 0.1)
    raw = rng.integers(0, n_v, n)
    raw[7777], raw[20001] = n_v + 5, n_v  # the first out-of-range valid index is named
    mask = np.zeros(n, bool)
    mask[100] = True
    raw[100] = n_v + 99                   # a null index is never checked
    idx = pa.array(raw, it, mask=mask)
    other = pa.array(rng.uniform(0, 1e6, n).astype(np.float32))
    dv, di, do = (DeviceArray.from_arrow(x, ctx) for x in (values, idx, other))
    with pytest.raises(pa.ArrowIndexError) as want:
        pc.take(values, idx)
    for fn in (lambda: bc.take(dv, di), lambda: bc.take_cast_arith(dv, di, pa.float32(), "add", do)):
        msgs = []
        for partition in ("1", "0"):
            with pytest.raises(pa.ArrowIndexError) as err:
                _run(monkeypatch, partition, 1, fn)
            msgs.append(str(err.value))
        assert msgs[0] == msgs[1] == str(want.value)


def test_fullsize_partitioned_equals_direct(ctx, monkeypatch):
    """the bench's shape and seed (1B rows unless B200_FULLSIZE_ROWS says otherwise), both paths compared on the device"""
    import gc

    import torch
    from bench import SEED as BENCH_SEED, _view, make_validity

    n = int(os.environ.get("B200_FULLSIZE_ROWS", "1000000000"))
    gc.collect()
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()
    free, _ = torch.cuda.mem_get_info()
    if free < 50 * n:
        pytest.skip(f"needs ~{50 * n >> 30} GiB of free device memory")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(BENCH_SEED)
    values_t = torch.rand(n, dtype=torch.float64, device="cuda", generator=gen) * 1e6
    vvalid_t, v_nulls = make_validity(torch, n, gen)
    idx_t = torch.randint(0, n, (n,), dtype=torch.int64, device="cuda", generator=gen)
    other_t = torch.rand(n, dtype=torch.float32, device="cuda", generator=gen) * 1e6
    ovalid_t, o_nulls = make_validity(torch, n, gen)
    torch.cuda.synchronize()
    values = DeviceArray.from_pointers(ctx, pa.float64(), n, values_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)
    indices = DeviceArray.from_pointers(ctx, pa.int64(), n, idx_t.data_ptr())
    other = DeviceArray.from_pointers(ctx, pa.float32(), n, other_t.data_ptr(), validity_ptr=ovalid_t.data_ptr(), null_count=o_nulls)

    def device_copy(arr, buf, count, typestr):
        return torch.as_tensor(_view(arr.buffers[buf].ptr, count, typestr, arr), device="cuda").clone()

    results = {}
    for partition in ("1", "0"):
        monkeypatch.setenv("B2_TAKE_PARTITION", partition)
        monkeypatch.delenv("B2_TAKE_PART_BAND_KB", raising=False)
        out = bc.take_cast_arith(values, indices, pa.float32(), "add", other)
        ctx.sync()
        torch.cuda.synchronize()
        results[partition] = (out.null_count, device_copy(out, 1, n, "<i4"), device_copy(out, 0, n // 8, "|u1"))
        torch.cuda.synchronize()
        del out
    assert results["1"][0] == results["0"][0]
    assert torch.equal(results["1"][2], results["0"][2])   # validity, every whole byte
    assert torch.equal(results["1"][1], results["0"][1])   # every slot's value, bit for bit
