"""A numpy restatement of the cumulative functions (kernels/vector_cumulative_ops.cc:67-203, Identity / Min / Max in
kernels/base_arithmetic_internal.h:678-775), written without pyarrow.compute.

  * row i is Op(x_i, Op(x_{i-1}, ... start)); integer sum / prod wrap; the default start is Identity<Op>: sum 0,
    prod 1, min numeric_limits<T>::max(), max numeric_limits<T>::min() (for floats the largest finite value and the
    smallest positive normal);
  * float min / max ignore NaN and return the newer value on a tie, so the sign of a zero follows the newest zero;
  * skip_nulls=True: a null row is null and leaves the state alone; otherwise every row from the first null on is
    null and is not combined;
  * *_checked over an integer type raises "overflow" when the exact prefix over the combined rows leaves the type;
  * the mean is sum += double(x); ++count; sum / count, the start ignored;
  * chunks are one column: the state carries from chunk to chunk and the output is one array.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

FUNCTIONS = ("cumulative_sum", "cumulative_sum_checked", "cumulative_prod", "cumulative_prod_checked",
             "cumulative_min", "cumulative_max", "cumulative_mean")
TYPES = (pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64(),
         pa.float32(), pa.float64())


class Overflow(Exception):
    """Invalid("overflow")"""


def default_start(name: str, t: pa.DataType):
    dt = np.dtype(t.to_pandas_dtype())
    if "sum" in name:
        return dt.type(0)
    if "prod" in name:
        return dt.type(1)
    info = np.finfo(dt) if dt.kind == "f" else np.iinfo(dt)
    if name == "cumulative_min":
        return dt.type(info.max)
    return dt.type(info.smallest_normal if dt.kind == "f" else info.min)


def _values(arr: pa.Array, dt) -> tuple[np.ndarray, np.ndarray]:
    """the values (0 under a null) and the validity of an array"""
    valid = np.ones(len(arr), bool) if arr.null_count == 0 else np.asarray(arr.is_valid().to_numpy(zero_copy_only=False))
    vals = np.asarray(arr.fill_null(0).to_numpy(zero_copy_only=False), dtype=dt) if len(arr) else np.zeros(0, dt)
    return vals, valid


def _extreme(name: str, x: np.ndarray, start) -> np.ndarray:
    """running min / max from start over x, the newest of equal values winning, NaN ignored"""
    seq = np.concatenate([np.array([start], x.dtype), x])
    if x.dtype.kind == "f":
        acc = (np.fmin if name == "cumulative_min" else np.fmax).accumulate(seq)
        # where the running extreme is zero, its sign is the newest zero's (every zero seen tied with it)
        idx = np.arange(len(seq))
        last_zero = np.maximum.accumulate(np.where(seq == 0, idx, 0))
        zero = acc == 0
        acc = np.where(zero, seq[last_zero], acc)
    else:
        acc = (np.minimum if name == "cumulative_min" else np.maximum).accumulate(seq)
    return acc[1:]


def _checked_overflows(name: str, x: np.ndarray, start) -> bool:
    info = np.iinfo(x.dtype)
    lo, hi = int(info.min), int(info.max)
    if "sum" in name:
        exact = np.cumsum(np.concatenate([[int(start)], x.astype(object)]))
        return bool(((exact < lo) | (exact > hi)).any())
    cur = int(start)
    for v in x.tolist():
        cur *= int(v)
        if not lo <= cur <= hi:
            return True
    return False


def cumulative(name: str, values, start=None, skip_nulls: bool = False) -> pa.Array:
    """name over a pa.Array, or a list of pa.Arrays taken as the chunks of one column; start: a Python number or
    numpy scalar of the input's type (the caller casts it), None for the default."""
    chunks = [values] if isinstance(values, pa.Array) else list(values)
    t = chunks[0].type
    dt = np.dtype(t.to_pandas_dtype())
    parts = [_values(c, dt) for c in chunks]
    x = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, dt)
    valid = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, bool)
    n = len(x)
    if skip_nulls:
        combined = valid.copy()
        out_valid = valid
    else:
        first = int(np.argmin(valid)) if not valid.all() else n
        combined = np.arange(n) < first
        out_valid = combined
    xs = x[combined]
    if name == "cumulative_mean":
        # the sum starts at +0.0, so a leading -0.0 gives +0.0
        acc = np.cumsum(np.concatenate([[0.0], xs.astype(np.float64)]))[1:] / np.arange(1, len(xs) + 1, dtype=np.float64)
        res = np.zeros(n, np.float64)
        res[combined] = acc
        return pa.array(res, pa.float64(), mask=~out_valid if not out_valid.all() else None)
    if isinstance(start, pa.Scalar):  # a null start contributes the value bits it carries: zero, as pyarrow builds it
        start = start.as_py() if start.is_valid else 0
    s = default_start(name, t) if start is None else dt.type(start)
    if name.endswith("_checked") and dt.kind != "f" and _checked_overflows(name, xs, s):
        raise Overflow("overflow")
    if name in ("cumulative_min", "cumulative_max"):
        acc = _extreme(name, xs, s)
    elif dt.kind == "f":
        seq = np.concatenate([np.array([s], dt), xs])
        with np.errstate(all="ignore"):
            acc = (np.cumsum(seq, dtype=dt) if "sum" in name else np.cumprod(seq, dtype=dt))[1:]
    else:  # two's complement: wrap modulo 2^64, then to the type's width
        seq = np.concatenate([np.array([s], dt), xs]).astype(np.uint64)
        with np.errstate(all="ignore"):
            acc = (np.cumsum(seq, dtype=np.uint64) if "sum" in name else np.cumprod(seq, dtype=np.uint64))[1:].astype(dt)
    res = np.zeros(n, dt)
    res[combined] = acc
    return pa.array(res, t, mask=~out_valid if not out_valid.all() else None)
