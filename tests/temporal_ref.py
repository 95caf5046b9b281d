"""Exact restatement of the temporal casts and calendar / clock fields (kernels/scalar_cast_temporal.cc,
kernels/scalar_temporal_unary.cc:222-691), without pyarrow.compute.

Values are numpy int64 arrays of the storage; arithmetic wraps as the reference's int / int64 expressions do.  The
reference reaches dates through the vendored date library, whose day count is a 32-bit int and whose year a 16-bit
short, so far-out values wrap:
  * floor<days>(t): trunc(t / day) narrowed to int32, then one day less when that day, scaled back to t's unit in
    wrapping int64, lies after t (so an exact multiple of a day far below 1970 still steps back one day);
  * civil-from-days over that day count in wrapping 32-bit int / unsigned arithmetic, the year truncated to 16 bits and
    the month and day to 8 bits.
Offset zones (UTC, "+HH:MM", "+HHMM", "-HH:MM", "-HHMM") shift the date fields, hour, minute and the timestamp ->
date / time casts to local time (ZonedLocalizer); the finer fields ignore the zone.
"""
from __future__ import annotations

import re

import numpy as np
import pyarrow as pa

PER_SECOND = {"s": 1, "ms": 1000, "us": 1000000, "ns": 1000000000}
M32 = 0xFFFFFFFF
DATE_FIELDS = ("year", "month", "day", "day_of_year", "day_of_week", "quarter", "is_leap_year")
CLOCK_FIELDS = ("hour", "minute", "second", "millisecond", "microsecond", "nanosecond", "subsecond")
FIELDS = DATE_FIELDS + CLOCK_FIELDS


def _i64(x) -> np.ndarray:
    return np.asarray(x, dtype=np.int64)


def wrap32(x) -> np.ndarray:
    """int32 two's-complement narrowing, widened back to int64"""
    return _i64(x).astype(np.int32).astype(np.int64)


def tdiv(a, b: int) -> np.ndarray:
    """C++ integer division (toward zero) of int64 a by a positive constant b"""
    a = _i64(a)
    r = np.mod(a, b)
    return a // b + ((r != 0) & (a < 0))


def tmod(a, b: int) -> np.ndarray:
    a = _i64(a)
    r = np.mod(a, b)
    return np.where((r != 0) & (a < 0), r - b, r)


def zone_offset(tz) -> int:
    """minutes east of UTC of a zone the device takes; None for a naive timestamp"""
    if tz is None or tz == "UTC":
        return 0
    m = re.fullmatch(r"([+-])(\d\d):?(\d\d)", tz)
    if m is None:
        raise ValueError(tz)
    v = int(m.group(2)) * 60 + int(m.group(3))
    return -v if m.group(1) == "-" else v


def unit_of(t: pa.DataType) -> str:
    if pa.types.is_date32(t):
        return "day"
    if pa.types.is_date64(t):
        return "ms"
    return t.unit


def shift_of(t: pa.DataType) -> int:
    if pa.types.is_timestamp(t) and t.tz is not None:
        return zone_offset(t.tz) * 60 * PER_SECOND[t.unit]
    return 0


def floor_days(t, per_day: int) -> np.ndarray:
    """floor<days>(t) as the reference's compiled code yields it: the narrowed quotient less one, where the step back
    from INT32_MIN is not narrowed again (the time-of-day paths see -2^31 - 1; the day-count paths narrow it)"""
    t = _i64(t)
    with np.errstate(over="ignore"):
        d = wrap32(tdiv(t, per_day))
        back = d * np.int64(per_day)
        return np.where(back > t, d - 1, d)


def civil(days):
    """(year, month, day) of 32-bit day counts"""
    z = wrap32(_i64(days) + 719468)
    era = tdiv(np.where(z >= 0, z, wrap32(z - 146096)), 146097)
    doe = (z - era * 146097) & M32
    yoe = ((doe - doe // 1460 + doe // 36524 - doe // 146096) & M32) // 365
    y = (yoe + era * 400) & M32
    doy = (doe - (365 * yoe + yoe // 4 - yoe // 100)) & M32
    mp = ((5 * doy + 2) & M32) // 153
    d = (doy - ((153 * mp + 2) & M32) // 5 + 1) & M32
    m = np.where(mp < 10, mp + 3, mp - 9) & M32
    year = ((y + (m <= 2)) & 0xFFFF).astype(np.uint16).astype(np.int16).astype(np.int64)
    return year, m & 0xFF, d & 0xFF


def days_before_year(year) -> np.ndarray:
    """the day count of year/jan/0"""
    y = _i64(year) - 1
    era = tdiv(np.where(y >= 0, y, y - 399), 400)
    yoe = y - era * 400
    doe = yoe * 365 + yoe // 4 - yoe // 100 + 305
    return wrap32(era * 146097 + doe - 719468)


def weekday(days) -> np.ndarray:
    """0 = Sunday .. 6 = Saturday"""
    z = _i64(days)
    u = z & M32
    return np.where(z >= -4, ((u + 4) & M32) % 7, u % 7)


def day_count(values, t: pa.DataType) -> np.ndarray:
    v = _i64(values)
    if pa.types.is_date32(t):
        return wrap32(v)
    per_day = 86400 * PER_SECOND[unit_of(t)]
    with np.errstate(over="ignore"):
        return wrap32(floor_days(v + np.int64(shift_of(t)), per_day))


def field_types(field: str):
    """the input type families a field accepts"""
    return ("date", "timestamp") if field in DATE_FIELDS else ("time", "timestamp")


def accepts(field: str, t: pa.DataType) -> bool:
    fam = ("date" if pa.types.is_date(t) else "time" if pa.types.is_time(t) else
           "timestamp" if pa.types.is_timestamp(t) else None)
    return fam in field_types(field)


def field(name: str, values, t: pa.DataType, week_start: int = 1, count_from_zero: bool = True) -> np.ndarray:
    """the field of every value (int64; float64 for subsecond; bool for is_leap_year)"""
    v = _i64(values)
    if name in DATE_FIELDS:
        d = day_count(v, t)
        if name == "day_of_week":
            iso = np.where(weekday(d) == 0, 7, weekday(d))
            r = iso - 1 + 8 - week_start
            r = np.where(r > 6, r - 7, r)
            return r + (0 if count_from_zero else 1)
        y, m, dd = civil(d)
        if name == "year":
            return y
        if name == "month":
            return m
        if name == "day":
            return dd
        if name == "quarter":
            return (m - 1) // 3 + 1
        if name == "day_of_year":
            return wrap32(d - days_before_year(y))
        return (tmod(y, 4) == 0) & ((tmod(y, 100) != 0) | (tmod(y, 400) == 0))
    s = PER_SECOND[t.unit]
    with np.errstate(over="ignore"):
        local = v + np.int64(shift_of(t))
        if name == "hour":
            per_day = 86400 * s
            rem = local - floor_days(local, per_day) * np.int64(per_day)
            return tdiv(rem, 3600 * s)
    if name == "minute":
        return np.mod(local, 3600 * s) // (60 * s)
    if name == "second":
        return np.mod(v, 60 * s) // s
    sub = np.mod(v, s)
    if name == "subsecond":
        return sub.astype(np.float64) / float(s)
    if name == "millisecond":
        return (sub // (s // 1000)) % 1000 if s >= 1000 else np.zeros_like(v)
    if name == "microsecond":
        return (sub // (s // 1000000)) % 1000 if s >= 1000000 else np.zeros_like(v)
    return sub % 1000 if s == 1000000000 else np.zeros_like(v)


# ---------------------------------------------------------------------------------------------------------------
# casts
# ---------------------------------------------------------------------------------------------------------------
class CastError(Exception):
    """the reference's Status::Invalid for a cast; str() is its message"""


def _kind(t: pa.DataType) -> str:
    for k, pred in (("date32", pa.types.is_date32), ("date64", pa.types.is_date64), ("time32", pa.types.is_time32),
                    ("time64", pa.types.is_time64), ("timestamp", pa.types.is_timestamp),
                    ("duration", pa.types.is_duration)):
        if pred(t):
            return k
    return str(t)  # int32 / int64


_UNITS = ("s", "ms", "us", "ns")


def _ratio(a: str, b: str) -> int:
    return PER_SECOND[a] // PER_SECOND[b]


def cast_plan(src: pa.DataType, dst: pa.DataType):
    """("shift", mul, factor) / ("ts_date",) / ("ts_time", mul, factor), or None when the reference has no kernel"""
    a, b = _kind(src), _kind(dst)

    def convert(fu, tu):
        return ("shift", True, _ratio(tu, fu)) if _UNITS.index(tu) >= _UNITS.index(fu) else ("shift", False, _ratio(fu, tu))

    if a == b and (a in ("date32", "date64", "int32", "int64") or src.unit == dst.unit):
        return ("shift", True, 1)
    if (a == "int32" and b in ("date32", "time32")) or (b == "int32" and a in ("date32", "time32")):
        return ("shift", True, 1)
    if (a == "int64" and b in ("date64", "time64", "timestamp", "duration")) or \
            (b == "int64" and a in ("date64", "time64", "timestamp", "duration")):
        return ("shift", True, 1)
    if (a, b) in (("timestamp", "timestamp"), ("duration", "duration")) or \
            (a in ("time32", "time64") and b in ("time32", "time64")):
        return convert(src.unit, dst.unit)
    if (a, b) == ("date32", "date64"):
        return ("shift", True, 86400000)
    if (a, b) == ("date64", "date32"):
        return ("shift", False, 86400000)
    if (a, b) == ("date32", "timestamp"):
        return ("shift", True, 86400 * PER_SECOND[dst.unit])
    if (a, b) == ("date64", "timestamp"):
        return convert("ms", dst.unit)
    if a == "timestamp" and b in ("date32", "date64"):
        return ("ts_date",)
    if a == "timestamp" and b in ("time32", "time64"):
        up = _UNITS.index(dst.unit) >= _UNITS.index(src.unit)
        return ("ts_time", up, _ratio(dst.unit, src.unit) if up else _ratio(src.unit, dst.unit))
    return None


def unsupported_message(src: pa.DataType, dst: pa.DataType) -> str:
    k = _kind(dst)
    return f"Unsupported cast from {src} to {k} using function cast_{k}"


def _narrow(x, dst: pa.DataType) -> np.ndarray:
    return wrap32(x) if dst.bit_width == 32 else _i64(x)


def cast(values, valid, src: pa.DataType, dst: pa.DataType, allow_time_truncate=False, allow_time_overflow=False):
    """(the output storage as int64, or raises CastError / NotImplementedError); only valid slots are checked and the
    first offending one is named"""
    plan = cast_plan(src, dst)
    if plan is None:
        raise NotImplementedError(unsupported_message(src, dst))
    v = _i64(values)
    valid = np.asarray(valid, bool)
    with np.errstate(over="ignore"):
        if plan[0] == "shift":
            _, mul, f = plan
            if mul:
                # INT64_MIN / f truncates toward zero
                lo = -((2 ** 63) // f)
                bad = ((v < lo) | (v > (2 ** 63 - 1) // f)) if f != 1 else np.zeros(len(v), bool)
                out = _narrow(v * np.int64(f), dst)
                if not allow_time_overflow:
                    _raise_first(bad & valid, v, f"Casting from {src} to {dst} would result in out of bounds timestamp")
                return out
            out = _narrow(tdiv(v, f), dst)
            if not allow_time_truncate:
                _raise_first((out * np.int64(f) != v) & valid, v, f"Casting from {src} to {dst} would lose data")
            return out
        local = v + np.int64(shift_of(src))
        per_day = 86400 * PER_SECOND[src.unit]
        d = floor_days(local, per_day)
        if plan[0] == "ts_date":
            # date64 from a finer unit sees the step back from INT32_MIN unnarrowed, as the time of day does; from
            # timestamp[s] it is narrowed (pyarrow 24's compiled code differs by unit)
            if pa.types.is_date32(dst) or src.unit == "s":
                d = wrap32(d)
            return d if pa.types.is_date32(dst) else d * np.int64(86400000)
        _, up, f = plan
        tod = local - d * np.int64(per_day)
        if up:
            return _narrow(tod * np.int64(f), dst)
        out = _narrow(tdiv(tod, f), dst)
        if not allow_time_truncate:
            # the extraction sets the status at every offending row and keeps going: the last one is named
            _raise_first(((out * np.int64(f) != tod) & valid)[::-1], tod[::-1], "Cast would lose data")
        return out


def _raise_first(bad: np.ndarray, shown: np.ndarray, text: str) -> None:
    idx = np.flatnonzero(bad)
    if len(idx):
        raise CastError(f"{text}: {int(shown[idx[0]])}")


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def type_variants():
    """every temporal type x unit, and the zone forms of timestamps"""
    out = [pa.date32(), pa.date64(), pa.time32("s"), pa.time32("ms"), pa.time64("us"), pa.time64("ns")]
    for u in _UNITS:
        out += [pa.timestamp(u), pa.timestamp(u, "UTC"), pa.timestamp(u, "+05:30"), pa.timestamp(u, "-0800"),
                pa.duration(u)]
    return out


def edge_values(t: pa.DataType) -> np.ndarray:
    """±0 and ±1 around midnight and 1970, leap days in 1900, 2000 and 2100, INT32 / INT64 min and max, and exact
    multiples of a day far below 1970"""
    import datetime as dt
    days = [0, -1, 1]
    for y, m, d in ((1900, 2, 28), (1900, 3, 1), (2000, 2, 29), (2000, 3, 1), (2100, 2, 28), (2100, 3, 1),
                    (1969, 12, 31), (1600, 2, 29), (9999, 12, 31), (1, 1, 1)):
        days.append((dt.date(y, m, d) - dt.date(1970, 1, 1)).days)
    i32 = [0, 1, -1, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 2, -2 ** 31 + 1]
    if t.bit_width == 32:
        per_day = 1 if pa.types.is_date32(t) else 86400 * PER_SECOND[getattr(t, "unit", "s")]
        vals = set(i32)
        for d in days:
            for e in (-1, 0, 1):
                x = d * per_day + e
                if -2 ** 31 <= x < 2 ** 31:
                    vals.add(x)
        return np.array(sorted(vals), np.int64)
    per_day = 86400 * PER_SECOND[unit_of(t) if t != pa.int64() else "s"]
    vals = set(i32) | {2 ** 63 - 1, -2 ** 63, 2 ** 63 - 2, -2 ** 63 + 1, 2 ** 62, -2 ** 62, 10 ** 12, -10 ** 12}
    for d in days + [-(2 ** 40), -(2 ** 33), 2 ** 33, -(2 ** 31) - 1, 2 ** 31]:
        for e in (-1, 0, 1):
            x = d * per_day + e
            if -2 ** 63 <= x < 2 ** 63:
                vals.add(x)
    return np.array(sorted(vals), np.int64)


def random_values(t: pa.DataType, n: int, seed: int) -> np.ndarray:
    """seeded full-range values of t's storage, half of them over every bit width"""
    rng = np.random.default_rng(seed)
    bits = t.bit_width
    full = rng.integers(-2 ** (bits - 1), 2 ** (bits - 1), n, dtype=np.int64, endpoint=False)
    widths = rng.integers(1, bits, n)
    narrow = rng.integers(-2 ** 62, 2 ** 62, n, dtype=np.int64) >> (63 - widths)
    return np.where(rng.random(n) < 0.5, full, narrow).astype(np.int64)


def to_arrow(values: np.ndarray, valid, t: pa.DataType) -> pa.Array:
    """an array of type t holding the storage values (and nulls where valid is false)"""
    storage = pa.array(_i64(values).astype(np.int32 if t.bit_width == 32 else np.int64),
                       mask=None if valid is None else ~np.asarray(valid, bool))
    return storage.view(t)
