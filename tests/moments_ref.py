"""numpy restatement of the reference's variance / stddev / skew / kurtosis, and exact Fraction references.

The reference (arrow/compute/kernels):
  * IntegerVarStd (aggregate_var_std_internal.h:33-57): int8..uint32 at level 2, one pass with exact integer sums;
    m2 = (square_sum - sum^2 // count) - (sum^2 % count) / count in double;
  * the two-pass per batch (aggregate_var_std.cc:106-131, hash_aggregate_numeric.cc:556-602): mean = sum / count, then
    sum((v - mean)^k) in double; integer sums are the accumulator type's (int64 / uint64, wrapping);
  * Moments::Merge (aggregate_var_std_internal.h:116-152) with NeumaierSum (util/math_internal.h:44-60);
  * Moments::Variance / Stddev / Skew / Kurtosis (:72-112) and the null rules of Finalize
    (hash_aggregate_numeric.cc:747-805, aggregate_var_std.cc:200-226).
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import pyarrow as pa

LEVEL = {"variance": 2, "stddev": 2, "skew": 3, "kurtosis": 4}
NARROW = {pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32()}


def neumaier(vals) -> float:
    s = c = 0.0
    for v in vals:
        t = s + v
        if math.isfinite(t):
            c += (s - t) + v if abs(s) >= abs(v) else (v - t) + s
        s = t
    return s + c


def batch_moments(vals: np.ndarray, t: pa.DataType, level: int):
    """(count, mean, m2, m3, m4) of one batch's valid values"""
    n = len(vals)
    if n == 0:
        return (0, 0.0, 0.0, 0.0, 0.0)
    if t in NARROW and level == 2:
        ints = [int(v) for v in vals]
        s, sq = sum(ints), sum(v * v for v in ints)
        ss = s * s
        m2 = float(sq - ss // n) - float(ss % n) / n
        return (n, float(s) / n, m2, 0.0, 0.0)
    if pa.types.is_floating(t):
        mean = float(np.sum(vals.astype(np.float64))) / n
    else:
        s = sum(int(v) for v in vals)
        s = s % (1 << 64)
        if pa.types.is_signed_integer(t) and s >= 1 << 63:
            s -= 1 << 64  # the int64 accumulator wraps
        mean = float(s) / n
    with np.errstate(all="ignore"):
        d = vals.astype(np.float64) - mean
        d2 = d * d
        return (n, mean, float(np.sum(d2)), float(np.sum(d2 * d)) if level >= 3 else 0.0,
                float(np.sum(d2 * d2)) if level >= 4 else 0.0)


def merge(level: int, a, b):
    if a[0] == 0:
        return b
    if b[0] == 0:
        return a
    na, ma, a2, a3, a4 = a
    nb, mb, b2, b3, b4 = b
    n = na + nb
    mean = (ma * na + mb * nb) / n
    m2 = neumaier([a2, b2, na * (ma - mean) * (ma - mean), nb * (mb - mean) * (mb - mean)])
    m3 = m4 = 0.0
    if level >= 3:
        delta = mb - ma
        delta2 = delta * delta
        m3 = neumaier([a3, b3, delta2 * delta * na * nb * (na - nb) / (n * n), 3 * delta * (na * b2 - nb * a2) / n])
        if level >= 4:
            m4 = neumaier([a4, b4, (delta2 * delta2) * na * nb * (na * na - na * nb + nb * nb) / (n * n * n),
                           6 * delta2 * (na * na * b2 + nb * nb * a2) / (n * n), 4 * delta * (na * b3 - nb * a3) / n])
    return (n, mean, m2, m3, m4)


def statistic(function: str, m, ddof=0, biased=True) -> float:
    n, _, m2, m3, m4 = m
    with np.errstate(all="ignore"):
        n, m2, m3, m4 = np.float64(n), np.float64(m2), np.float64(m3), np.float64(m4)
        if function in ("variance", "stddev"):
            v = m2 / (n - ddof)
            return float(np.sqrt(v) if function == "stddev" else v)
        if function == "skew":
            if biased:
                return float(np.sqrt(n) * m3 / np.sqrt(m2 * m2 * m2))
            a = m2 / n
            return float(np.sqrt(n * (n - 1)) / (n - 2) * (m3 / n) / np.sqrt(a * a * a))
        if biased:
            return float(n * m4 / (m2 * m2) - 3)
        a = m2 / n
        return float(1.0 / ((n - 2) * (n - 3)) * ((n * n - 1.0) * (m4 / n) / (a * a) - 3 * ((n - 1) * (n - 1))))


def is_null(function: str, count: int, saw_null: bool, ddof=0, skip_nulls=True, min_count=0, biased=True) -> bool:
    d = ddof if function in ("variance", "stddev") else 0
    return (count <= d or count < min_count or (not skip_nulls and saw_null)
            or (function == "skew" and not biased and count < 3) or (function == "kurtosis" and not biased and count < 4))


def _valid(arr: pa.Array) -> np.ndarray:
    return np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)


def scalar(function: str, chunks, ddof=0, skip_nulls=True, min_count=0, biased=True):
    """the ungrouped statistic over a list of chunks (one batch each), None for null"""
    level, m, saw_null = LEVEL[function], (0, 0.0, 0.0, 0.0, 0.0), False
    for c in chunks:
        ok = _valid(c)
        saw_null |= not ok.all()
        vals = np.asarray(c.to_numpy(zero_copy_only=False))[ok] if len(c) else np.zeros(0)
        m = merge(level, m, batch_moments(vals.astype(c.type.to_pandas_dtype()), c.type, level))
    if is_null(function, m[0], saw_null, ddof, skip_nulls, min_count, biased):
        return None
    return statistic(function, m, ddof, biased)


def grouped(function: str, batches, num_groups: int, ddof=0, skip_nulls=True, min_count=0, biased=True):
    """per-group statistic over batches [(values pa.Array, ids np.ndarray)], a list with None for null groups"""
    level = LEVEL[function]
    state = [(0, 0.0, 0.0, 0.0, 0.0)] * num_groups
    saw = [False] * num_groups
    for vals, ids in batches:
        ok = _valid(vals)
        raw = np.asarray(vals.to_numpy(zero_copy_only=False))
        for g in range(num_groups):
            sel = ids == g
            if (~ok[sel]).any():
                saw[g] = True
            v = raw[sel & ok].astype(vals.type.to_pandas_dtype())
            state[g] = merge(level, state[g], batch_moments(v, vals.type, level))
    return [None if is_null(function, state[g][0], saw[g], ddof, skip_nulls, min_count, biased)
            else statistic(function, state[g], ddof, biased) for g in range(num_groups)]


# ---- exact references ----
def exact_variance(vals, ddof=0) -> Fraction:
    """N / D with N = n * sum(x^2) - sum(x)^2, D = n * (n - ddof): the population moment, exactly"""
    xs = [int(v) for v in vals]
    n = len(xs)
    return Fraction(n * sum(x * x for x in xs) - sum(xs) ** 2, n * (n - ddof))


def exact_central(vals, k: int) -> Fraction:
    """sum((x - mean)^k) with the exact mean of the values (ints or floats, each exact as a Fraction)"""
    xs = [Fraction(float(v)) if isinstance(v, (float, np.floating)) else Fraction(int(v)) for v in vals]
    mu = sum(xs) / len(xs)
    return sum((x - mu) ** k for x in xs)


def exact_statistic(function: str, vals, ddof=0, biased=True) -> float:
    """the statistic computed from exact central moments, rounded once per step only where a sqrt is needed"""
    n = len(vals)
    if function in ("variance", "stddev"):
        v = exact_central(vals, 2) / (n - ddof)
        return math.sqrt(v) if function == "stddev" else float(v)
    m2, m3, m4 = exact_central(vals, 2), exact_central(vals, 3), exact_central(vals, 4)
    if function == "skew":
        g = float(m3 / n) / math.sqrt(float(m2 / n)) ** 3
        return g if biased else g * math.sqrt(n * (n - 1)) / (n - 2)
    if biased:
        return float(Fraction(n) * m4 / (m2 * m2) - 3)
    a = m2 / n
    return float(Fraction(1, (n - 2) * (n - 3)) * ((n * n - 1) * (m4 / n) / (a * a) - 3 * (n - 1) ** 2))


def tolerance(function: str, vals, c: float = 16.0) -> float:
    """|got - exact| bound of the two-pass in double, relative to the result: per moment k used,
    c * n * 2^-53 * sum|x - mu|^k / |sum (x - mu)^k|, plus the mean's rounding carried through the k-th power,
    c * n * 2^-53 * k * (|mu| + max|x - mu|) * sum|x - mu|^(k-1) / |sum (x - mu)^k|.
    Within ONE batch that term cancels at k = 2 (sum (x - mu) = 0), but the device and the reference both consume in
    batches (Acero cuts 32Ki-row batches) and combine them with Moments::Merge, whose terms n_j * (mean_j - mean)^2 take
    each batch mean with its own rounding error (up to n_j * 2^-53 * (|mu| + max|x - mu|) from a naive sum): to first
    order 2 * sum_j n_j * |mean_j - mean| * that error, which the k = 2 term bounds.  Measured on data offset 1e12 from
    zero, both the reference and the device exceed the bound without it by up to 40x."""
    x = np.asarray(vals, dtype=np.float64)
    n = len(x)
    mu = float(np.mean(x))
    d = np.abs(x - mu)
    eps = 2.0 ** -53
    rel = 0.0
    for k in range(2, LEVEL[function] + 1):
        den = abs(float(exact_central(vals, k))) if k > 2 else float(np.sum(d ** 2))
        if den == 0:
            return math.inf
        mean_term = k * (abs(mu) + float(np.max(d))) * n * float(np.sum(d ** (k - 1)))
        rel += (n * float(np.sum(d ** k)) + mean_term) / den
    return c * eps * rel


def tolerance_abs(function: str, vals, c: float = 16.0) -> float:
    """the bound of tolerance() as an absolute error of the statistic, usable where the statistic is 0 (a symmetric group's
    skew): each moment's error dm_k (as in tolerance) times the statistic's first-order sensitivity to m_k and m2"""
    x = np.asarray(vals, dtype=np.float64)
    n = len(x)
    mu = float(np.mean(x))
    d = np.abs(x - mu)
    s = {k: float(np.sum(d ** k)) for k in range(1, 5)}
    if s[2] == 0:
        return 0.0
    eps = 2.0 ** -53
    dm = {k: c * eps * n * (s[k] + k * (abs(mu) + float(np.max(d))) * s[k - 1]) for k in (2, 3, 4)}
    m = {k: float(exact_central(vals, k)) for k in (2, 3, 4)} if function in ("skew", "kurtosis") else {2: s[2]}
    unbiased = max(1.0, math.sqrt(n * (n - 1)) / (n - 2) if n > 2 else 1.0, (n * n - 1.0) / ((n - 2) * (n - 3)) if n > 3 else 1.0)
    if function == "variance":
        return dm[2] / max(n - 1, 1)
    if function == "stddev":
        return dm[2] / max(n - 1, 1) / math.sqrt(s[2] / n)
    if function == "skew":
        return unbiased * math.sqrt(n) / s[2] ** 1.5 * (dm[3] + 1.5 * abs(m[3]) * dm[2] / s[2])
    return unbiased * n / s[2] ** 2 * (dm[4] + 2 * abs(m[4]) * dm[2] / s[2]) + 3 * unbiased * dm[2] / s[2]
