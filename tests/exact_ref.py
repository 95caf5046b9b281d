"""Exact references for aggregation and hashing tests, and the rule results are compared by.

- Integer sums: exact Python integers, reduced mod 2^64 into the accumulator type (int64 / uint64 wrap like the reference).
- Float sums: math.fsum, or exact integer sums for integer-valued floats.
- Rows are aligned by the BITS of the key (an unsigned integer of the key's width), never by its value: sorting by value
  cannot order -0.0 against +0.0 or tell NaN payloads apart, and the kernels group by bytes.
- Comparison: bit-exact, except that any NaN equals any NaN and, for min / max only, -0.0 equals +0.0 (the reference keeps
  whichever zero it sees first: min_max([-0.0, 0.0]) is -0.0 / -0.0, min_max([0.0, -0.0]) is 0.0 / 0.0)."""
import math

import numpy as np
import pyarrow as pa

UINT_OF_WIDTH = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}

# special float bit patterns, as unsigned integers of the float's width
F64_SPECIAL = {
    "+0": 0x0000000000000000, "-0": 0x8000000000000000, "qnan": 0x7FF8000000000000, "-qnan": 0xFFF8000000000000,
    "nan_payload": 0x7FF800000000BEEF, "snan": 0x7FF0000000000001, "all_ones": 0xFFFFFFFFFFFFFFFF,
    "+inf": 0x7FF0000000000000, "-inf": 0xFFF0000000000000, "min_denormal": 0x0000000000000001,
}
F32_SPECIAL = {
    "+0": 0x00000000, "-0": 0x80000000, "qnan": 0x7FC00000, "-qnan": 0xFFC00000, "nan_payload": 0x7FC0BEEF,
    "snan": 0x7F800001, "all_ones": 0xFFFFFFFF, "+inf": 0x7F800000, "-inf": 0xFF800000, "min_denormal": 0x00000001,
}


def special_values(dtype) -> np.ndarray:
    """the special keys / values of the float dtype, one each"""
    dtype = np.dtype(dtype)
    table = F32_SPECIAL if dtype.itemsize == 4 else F64_SPECIAL
    return np.array(list(table.values()), dtype=UINT_OF_WIDTH[dtype.itemsize]).view(dtype)


GROUP_CLASSES = ("all_nan", "nan_and_finite", "pos_inf", "both_inf", "neg_zero", "mixed_zero", "denormal", "all_null",
                 "few_values", "finite")


def special_float_groups(dtype, num_groups: int, n: int, seed: int, null_probability=0.1):
    """(ids uint32, values) with group g of class GROUP_CLASSES[g % 10]; every group has rows, "few_values" groups at most
    two valid values (empty after min_count = 3).  Finite values are signed powers of two in [0.5, 4] and denormals are
    powers of two below 2^20 units in the last place, so every sum, mean and product is exact in double in ANY order: the
    result does not depend on how a kernel orders its additions."""
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    ids = (np.arange(n) % num_groups).astype(np.uint32)
    rng.shuffle(ids)
    cls = ids % len(GROUP_CLASSES)
    sp = dict(zip((F32_SPECIAL if dtype.itemsize == 4 else F64_SPECIAL).keys(), special_values(dtype)))
    finite = rng.choice(np.array([0.5, 1, 2, 4, -0.5, -1, -2, -4], dtype=dtype), n)
    # quiet NaNs only: std::fmin / fmax turn a signalling NaN into a quiet NaN that replaces the running min / max, so
    # with one in a group the reference's hash_min / hash_max depend on row order (signalling NaNs are tested as keys)
    nans = rng.choice(np.array([sp["qnan"], sp["-qnan"], sp["nan_payload"], sp["all_ones"]], dtype=dtype), n)
    tiny = np.ldexp(np.ones(n), rng.integers(0, 20, n) + (-149 if dtype.itemsize == 4 else -1074)).astype(dtype)
    v = finite.copy()
    v[cls == 0] = nans[cls == 0]
    half = rng.random(n) < 0.35
    v[(cls == 1) & half] = nans[(cls == 1) & half]
    v[cls == 2] = sp["+inf"]
    v[cls == 3] = np.where(half, sp["-inf"], sp["+inf"])[cls == 3]
    v[cls == 4] = sp["-0"]
    v[cls == 5] = np.where(half, sp["-0"], sp["+0"])[cls == 5]
    v[cls == 6] = tiny[cls == 6]
    null = rng.random(n) < null_probability
    null |= cls == 7
    # "few_values": the first two rows of the group stay, later ones are null
    order = np.argsort(ids, kind="stable")
    rank = np.empty(n, np.int64)
    starts = np.searchsorted(ids[order], ids[order])
    rank[order] = np.arange(n) - starts
    null |= (cls == 8) & (rank >= 2)
    return ids, pa.array(v, mask=null)


def raw(arr: pa.Array) -> np.ndarray:
    """the value buffer of a fixed-width array as numpy, null slots included (whatever bits they hold)"""
    t = arr.type
    dt = np.dtype(t.to_pandas_dtype())
    buf = arr.buffers()[1]
    return np.frombuffer(buf, dtype=dt, count=arr.offset + len(arr))[arr.offset:] if buf is not None else np.zeros(len(arr), dt)


def valid_mask(arr: pa.Array) -> np.ndarray:
    return np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)


def bits(arr_or_np) -> np.ndarray:
    """values viewed as unsigned integers of their own width"""
    v = raw(arr_or_np) if isinstance(arr_or_np, pa.Array) else np.ascontiguousarray(arr_or_np)
    return v.view(UINT_OF_WIDTH[v.dtype.itemsize])


def key_order(keys: pa.Array) -> np.ndarray:
    """row permutation that sorts by the key's bits, null keys last"""
    return np.lexsort((bits(keys), ~valid_mask(keys)))


def exact_int_sums(ids: np.ndarray, vals: np.ndarray, num_groups: int) -> list:
    """per-group sums of integer values as exact Python ints: 32-bit halves summed in 64 bits (no overflow below 2^31 rows
    per group), then recombined"""
    v = vals.astype(np.int64) if np.issubdtype(vals.dtype, np.signedinteger) else vals.astype(np.uint64)
    lo = (v.view(np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.uint64)
    hi = v >> (np.int64(32) if v.dtype == np.int64 else np.uint64(32))
    slo = np.zeros(num_groups, np.uint64)
    shi = np.zeros(num_groups, hi.dtype)
    np.add.at(slo, ids, lo)
    np.add.at(shi, ids, hi)
    return [int(h) * (1 << 32) + int(l) for h, l in zip(shi.tolist(), slo.tolist())]


def wrap64(x: int, signed: bool) -> int:
    """x reduced mod 2^64 into int64 (signed) or uint64"""
    x &= (1 << 64) - 1
    return x - (1 << 64) if signed and x >= (1 << 63) else x


def fsums(ids: np.ndarray, vals: np.ndarray, num_groups: int) -> list:
    """per-group math.fsum (the correctly rounded exact sum) of float values"""
    order = np.argsort(ids, kind="stable")
    bounds = np.searchsorted(ids[order], np.arange(num_groups + 1))
    sv = vals[order].astype(np.float64).tolist()
    return [math.fsum(sv[bounds[g]:bounds[g + 1]]) for g in range(num_groups)]


def count_distinct(ids: np.ndarray, vals: pa.Array, num_groups: int, mode="only_valid") -> np.ndarray:
    """hash_count_distinct: distinct (value BITS, group) pairs per group; a null is one more value under "all" """
    ok = valid_mask(vals)
    b = bits(vals).astype(np.uint64)
    sel = ok if mode == "only_valid" else (~ok if mode == "only_null" else np.ones(len(ids), bool))
    b = np.where(ok, b, 0)
    pairs = np.unique(np.stack([ids[sel].astype(np.uint64), b[sel], ok[sel].astype(np.uint64)], axis=1), axis=0)
    return np.bincount(pairs[:, 0].astype(np.int64), minlength=num_groups).astype(np.int64)


def same_value(a, b, zeros_equal=False) -> bool:
    """the comparison rule for two valid Python / numpy scalars"""
    if isinstance(a, float) or isinstance(b, float) or np.issubdtype(type(a), np.floating):
        a, b = float(a), float(b)
        if math.isnan(a) or math.isnan(b):
            return math.isnan(a) and math.isnan(b)
        if a == 0.0 and b == 0.0 and not zeros_equal:
            return math.copysign(1.0, a) == math.copysign(1.0, b)
        return a == b
    return a == b


def mismatches(got: pa.Array, want: pa.Array, zeros_equal=False) -> np.ndarray:
    """indices where got and want differ under the comparison rule (validity, then the bits of valid slots)"""
    assert got.type == want.type, f"type {got.type} != {want.type}"
    assert len(got) == len(want), f"length {len(got)} != {len(want)}"
    gv, wv = valid_mask(got), valid_mask(want)
    bad = gv != wv
    both = gv & wv
    gr, wr = raw(got), raw(want)
    if np.issubdtype(gr.dtype, np.floating):
        gb, wb = bits(gr), bits(wr)
        ok = (gb == wb) | (np.isnan(gr) & np.isnan(wr))
        if zeros_equal:
            ok |= (gr == 0) & (wr == 0)
        bad |= both & ~ok
    else:
        bad |= both & (gr != wr)
    return np.flatnonzero(bad)


def assert_same(got: pa.Array, want: pa.Array, zeros_equal=False, msg=""):
    if isinstance(got, pa.ChunkedArray):
        got = got.combine_chunks()
    if isinstance(want, pa.ChunkedArray):
        want = want.combine_chunks()
    bad = mismatches(got, want, zeros_equal)
    if len(bad):
        i = bad[:5].tolist()
        raise AssertionError(f"{msg}: {len(bad)} of {len(got)} differ, at {i}: got {[got[j] for j in i]} "
                             f"(bits {[hex(int(x)) for x in bits(got)[i]] if pa.types.is_floating(got.type) else ''}) "
                             f"want {[want[j] for j in i]}")
