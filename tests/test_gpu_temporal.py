"""Temporal casts and calendar / clock fields on the device (csrc/scalar_temporal.cu) against the restatement
(temporal_ref) and pyarrow.compute, compared under valid slots: every field x type x unit x zone form, every cast pair x
safety flag with its error text, nulls, slices at offsets that are not byte-aligned, lengths around the 32-row groups,
the refusals, one launch per call, and a 2^30 + k-row year / hour counted against a torch restatement."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import temporal_ref as ref
from tests.test_temporal_oracle import CAST_TYPES, TYPES, inputs

pytestmark = pytest.mark.gpu


def _storage(arr: pa.Array, t: pa.DataType) -> np.ndarray:
    st = pa.int32() if t.bit_width == 32 else pa.int64()
    return np.asarray(arr.view(st).fill_null(0))


def _valid(arr: pa.Array) -> np.ndarray:
    return np.asarray(arr.is_valid())


def check_field(ctx, field, arr: pa.Array, values: np.ndarray, valid: np.ndarray, **opts):
    got = getattr(bc, field)(DeviceArray.from_arrow(arr, ctx), **opts).to_arrow()
    assert len(got) == len(arr) and np.array_equal(_valid(got), valid), field
    want = ref.field(field, values, arr.type, **opts)
    g = got.fill_null(False if field == "is_leap_year" else 0).to_numpy(zero_copy_only=False)
    np.testing.assert_array_equal(g[valid], np.asarray(want, g.dtype)[valid], err_msg=f"{field} {arr.type}")
    return got


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_fields(ctx, t):
    v = inputs(t)
    rng = np.random.default_rng(3)
    valid = rng.random(len(v)) < 0.9
    arr = ref.to_arrow(v, valid, t)
    for field in ref.FIELDS:
        if not ref.accepts(field, t):
            with pytest.raises(pa.ArrowNotImplementedError, match=f"Function '{field}' has no kernel"):
                getattr(bc, field)(DeviceArray.from_arrow(arr, ctx))
            continue
        got = check_field(ctx, field, arr, v, valid)
        assert got.equals(pc.call_function(field, [arr])), (field, t)


@pytest.mark.parametrize("t", [pa.date32(), pa.timestamp("ms", "-08:00"), pa.timestamp("us")], ids=str)
def test_day_of_week_options(ctx, t):
    v = inputs(t, 300)
    arr = ref.to_arrow(v, None, t)
    for ws in range(1, 8):
        for cfz in (True, False):
            got = bc.day_of_week(DeviceArray.from_arrow(arr, ctx), count_from_zero=cfz, week_start=ws).to_arrow()
            assert got.equals(pc.day_of_week(arr, count_from_zero=cfz, week_start=ws))
            opts = pc.DayOfWeekOptions(count_from_zero=cfz, week_start=ws)
            assert bc.call_function("day_of_week", [DeviceArray.from_arrow(arr, ctx)], opts).to_arrow().equals(got)
    for ws in (0, 8):
        with pytest.raises(pa.ArrowInvalid, match=f"week_start must follow ISO convention .* Got week_start={ws}"):
            bc.day_of_week(DeviceArray.from_arrow(arr, ctx), week_start=ws)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 63, 64, 65, 1000, 4099])
@pytest.mark.parametrize("offset", [0, 3, 37])
def test_lengths_and_slices(ctx, n, offset):
    t = pa.timestamp("us", "+05:30")
    v = ref.random_values(t, n + offset + 5, n)
    valid = np.random.default_rng(n).random(len(v)) < 0.8
    full = ref.to_arrow(v, valid, t)
    dv = DeviceArray.from_arrow(full, ctx).slice(offset, n)
    part = full.slice(offset, n)
    for field in ("year", "is_leap_year", "hour", "subsecond"):
        got = getattr(bc, field)(dv).to_arrow()
        assert got.equals(pc.call_function(field, [part])), (field, n, offset)


def _cast(ctx, arr: pa.Array, src, dst, truncate, overflow):
    da = DeviceArray.from_arrow(arr, ctx)
    cin, cout = da._c(), _cabi.B2Array()
    f, t = bc.temporal_type(src), bc.temporal_type(dst)
    st = ctx.lib.b2_cast_temporal(ctx.handle, C.byref(cin), C.byref(f), C.byref(t), int(truncate), int(overflow),
                                  C.byref(cout), ctx.stream)
    if st != 0:
        return None, (st, _cabi.last_error())
    return DeviceArray._from_c(ctx, cout, dst).to_arrow(), None


def _device_text(text: str) -> str:
    """the device writes a zone from its offset: -0800 as -08:00"""
    return text.replace("tz=-0800", "tz=-08:00")


@pytest.mark.parametrize("src", CAST_TYPES, ids=str)
def test_casts(ctx, src):
    v = inputs(src, 300, 9)
    valid = np.random.default_rng(9).random(len(v)) < 0.9
    arr = ref.to_arrow(v, valid, src)
    for dst in CAST_TYPES:
        if src == dst or (src in (pa.int32(), pa.int64()) and dst in (pa.int32(), pa.int64())):
            continue
        for truncate, overflow in ((False, False), (True, False), (False, True), (True, True)):
            got, err = _cast(ctx, arr, src, dst, truncate, overflow)
            try:
                want = ref.cast(v, valid, src, dst, truncate, overflow)
            except ref.CastError as e:
                assert err == (_cabi.INVALID, _device_text(str(e))), (src, dst, truncate, overflow)
                continue
            except NotImplementedError as e:
                assert err == (_cabi.NOT_IMPLEMENTED, _device_text(str(e))), (src, dst)
                continue
            assert err is None, (src, dst, truncate, overflow, err)
            assert np.array_equal(_valid(got), valid)
            np.testing.assert_array_equal(_storage(got, dst)[valid], want[valid], err_msg=f"{src} -> {dst}")
            opts = pc.CastOptions(dst, allow_time_truncate=truncate, allow_time_overflow=overflow)
            w = pc.cast(arr, options=opts)
            np.testing.assert_array_equal(_storage(got, dst)[valid], _storage(w, dst)[valid])


def test_cast_error_names_first_valid_row(ctx):
    """a null slot is never checked; the first valid offending row is named (ShiftTime), the last for timestamp ->
    time (the extraction keeps going)"""
    ms = pa.timestamp("ms")
    arr = pa.array([1500, 2500, 1000, 3700], ms, mask=np.array([True, False, False, False]))
    _, err = _cast(ctx, arr, ms, pa.timestamp("s"), False, False)
    assert err == (_cabi.INVALID, "Casting from timestamp[ms] to timestamp[s] would lose data: 2500")
    _, err = _cast(ctx, arr, ms, pa.time32("s"), False, False)
    assert err == (_cabi.INVALID, "Cast would lose data: 3700")
    ok = pa.array([1500, 2000], ms, mask=np.array([True, False]))
    got, err = _cast(ctx, ok, ms, pa.timestamp("s"), False, False)
    assert err is None and got.cast(pa.int64()).to_pylist() == [None, 2]
    got, _ = _cast(ctx, pa.array([-1500, 1500], ms), ms, pa.timestamp("s"), True, False)
    assert got.cast(pa.int64()).to_pylist() == [-1, 1]
    _, err = _cast(ctx, pa.array([0, 2 ** 62], pa.int64()).view(pa.timestamp("s")), pa.timestamp("s"),
                   pa.timestamp("ns"), False, False)
    assert err == (_cabi.INVALID, f"Casting from timestamp[s] to timestamp[ns] would result in out of bounds timestamp: {2 ** 62}")


def test_named_zone_refused(ctx):
    arr = pa.array([0, 1], pa.timestamp("s", "America/New_York"))
    with pytest.raises(pa.ArrowNotImplementedError, match="America/New_York"):
        bc.year(DeviceArray.from_arrow(arr, ctx))
    with pytest.raises(pa.ArrowNotImplementedError, match="America/New_York"):
        bc.temporal_type(arr.type)


def test_python_cast_still_refuses_temporal(ctx):
    arr = pa.array([0, 1], pa.timestamp("ms"))
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.cast(DeviceArray.from_arrow(arr, ctx), pa.timestamp("s"))


def test_one_launch_per_call(ctx):
    t = pa.timestamp("us", "+05:30")
    arr = ref.to_arrow(ref.random_values(t, 100000, 1), None, t)
    dv = DeviceArray.from_arrow(arr, ctx)
    lib = ctx.lib
    for field in ref.FIELDS:
        before = lib.b2_launch_count()
        getattr(bc, field)(dv)
        assert lib.b2_launch_count() - before == 1, field
    for dst, truncate in ((pa.date32(), False), (pa.timestamp("ms"), True), (pa.time64("us"), False),
                          (pa.timestamp("ns"), False)):
        before = lib.b2_launch_count()
        _cast(ctx, arr, t, dst, truncate, False)
        assert lib.b2_launch_count() - before == 1, dst


def test_more_than_2_30_rows(ctx):
    """2^30 + 4099 timestamp[us] rows: year and hour against a torch restatement of the same arithmetic"""
    torch = pytest.importorskip("torch")
    n = (1 << 30) + 4099
    g = torch.Generator(device="cuda").manual_seed(7)
    # 1900 .. 2100 in microseconds, where the day count never wraps
    lo, hi = -2208988800 * 10 ** 6, 4102444800 * 10 ** 6
    t = torch.randint(lo, hi, (n,), dtype=torch.int64, device="cuda", generator=g)
    torch.cuda.synchronize()
    dv = DeviceArray.from_pointers(ctx, pa.timestamp("us"), n, t.data_ptr(), keepalive=t)
    per_day = 86400 * 10 ** 6
    chunk = 1 << 28
    for name in ("year", "hour"):
        got = getattr(bc, name)(dv)
        assert len(got) == n and got.null_count == 0
        mismatches = 0
        for start in range(0, n, chunk):
            c = t[start:start + chunk]
            days = torch.div(c, per_day, rounding_mode="floor")
            if name == "hour":
                want = torch.div(c - days * per_day, 3600 * 10 ** 6, rounding_mode="floor")
            else:
                z = days + 719468
                era = torch.div(z, 146097, rounding_mode="floor")
                doe = z - era * 146097
                yoe = torch.div(doe - doe // 1460 + doe // 36524 - doe // 146096, 365, rounding_mode="floor")
                doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
                want = yoe + era * 400 + ((5 * doy + 2) // 153 >= 10).to(torch.int64)
                del z, era, doe, yoe, doy
            torch.cuda.synchronize()
            m = len(c)
            dw = DeviceArray.from_pointers(ctx, pa.int64(), m, want.data_ptr(), keepalive=want)
            diff = bc.not_equal(got.slice(start, m), dw)
            cnt = C.c_int64()
            assert ctx.lib.b2_bitmap_count(ctx.handle, C.c_void_p(diff._c().data), 0, m, C.byref(cnt), ctx.stream) == 0
            mismatches += cnt.value
            del diff, dw, want, days
        assert mismatches == 0, name
        del got


def test_reference_expected_outputs(ctx):
    """the device reproduces the field outputs of the reference's own tests (tests/golden/kat_temporal.json)"""
    import json
    import os
    kat = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_temporal.json")))
    f = kat["fields"]
    times = pa.array([None if s is None else np.datetime64(s.replace(" ", "T"), "ns") for s in f["times"]], pa.timestamp("ns"))
    dv = DeviceArray.from_arrow(times, ctx)
    for name, want in f["expected"].items():
        got = getattr(bc, name)(dv).to_arrow().to_pylist()
        assert got == want, name
