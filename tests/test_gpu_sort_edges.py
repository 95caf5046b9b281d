"""sort_indices, sort_payload, the multi-key sort, select_k_unstable and the range kernels of the distributed sort against
the EXACT total-order references of tests/sort_ref.py (pinned to the reference binary by test_sort_edges_oracle.py), at
the places where a radix sort goes wrong:

- values: full-range integers and float bit patterns, NaNs of both signs and several payloads, +-0, +-inf, subnormals;
- sizes: row counts n and valid counts nv at k * tile +- 1 for both the prepare tiles (over n rows) and the one-sweep
  tiles (over nv keys), a last tile with fewer keys than one warp holds, nv = 0 and 1, and ~3 M keys (several waves of
  one-sweep CTAs chained by the decoupled look-back);
- skipped passes: data whose digits are constant except at chosen bytes, so the pass list sort_typed builds has one
  LAST pass, gaps between two passes, or no pass at all (the row numbers are widened directly);
- select_k's branches, restated from select_k.cu and asserted per case, so that the threshold path and each fallback
  are actually reached;
- the 2^30-row boundary of the look-back cells and the 2^32-row refusal.

Kernel constants are read from the sources, so the lengths follow the code."""
import ctypes as C
import os
import re

import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from arrow_b200 import _cabi as cabi
from arrow_b200.device import check
from tests import exact_ref as er
from tests import sort_ref as sr
from tests.util import SEED

pytestmark = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constant(text, name):
    m = re.search(rf"constexpr (?:int|int64_t) {name} = (\d+)(?: << (\d+))?;", text)
    return int(m.group(1)) << int(m.group(2) or 0)


_SORT, _SELECT, _PART = _source("sort_indices.cu"), _source("select_k.cu"), _source("partition.cu")
SORT_THREADS, SORT_ITEMS = _constant(_SORT, "kSortThreads"), _constant(_SORT, "kSortItems")
TILE = SORT_THREADS * SORT_ITEMS                       # keys per one-sweep tile
WARP_KEYS = 32 * SORT_ITEMS                            # keys of one warp's segment of a tile
PREP_TILE = _constant(_source("selection.cuh"), "kTileRows")   # rows per prepare (null partition) tile
SORT_LIMIT = (1 << 32) - int(re.search(r"if \(n >= \(1ll << 32\) - (\d+)\)", _SORT).group(1))
SAMPLE = _constant(_SELECT, "kSample")
_sw = re.search(r"if \(n < \(1 << (\d+)\) \|\| k \* (\d+) > n \|\|", _SELECT)
SELECT_MIN_N, SELECT_K_FACTOR = 1 << int(_sw.group(1)), int(_sw.group(2))
SPLIT_MAX = _constant(_PART, "kSplitMaxBins") - 2      # splitters of b2_range_split
PARTITION_MAX = int(re.search(r"splitters->length > (\d+)\) return set_error\(B2_INVALID, \"at most", _PART).group(1))
ORDER_ID = {"ascending": 0, "descending": 1}


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


def indices(d: DeviceArray) -> np.ndarray:
    a = d.to_arrow()
    assert a.type == pa.uint64() and a.null_count == 0
    return a.to_numpy().astype(np.int64)


def reference(arr, order, placement) -> np.ndarray:
    """the sorted form for small inputs, the vectorised one (pinned to it on the CPU) for large ones"""
    if len(arr) <= 20000:
        return np.array(sr.sort_indices_ref(arr, order, placement), np.int64)
    return sr.sort_indices_np(arr, order, placement)


def assert_sorted_like(got: np.ndarray, want: np.ndarray, msg):
    assert len(got) == len(want), f"{msg}: length {len(got)} != {len(want)}"
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, f"{msg}: {len(bad)} of {len(got)} rows differ, first at {bad[:5].tolist()}: " \
                          f"got {got[bad[:5]].tolist()} want {want[bad[:5]].tolist()}"


def exact_nulls(n, nv, rng) -> np.ndarray:
    """validity with exactly nv valid rows among n"""
    valid = np.zeros(n, bool)
    valid[rng.choice(n, nv, replace=False)] = True
    return valid


def unknown_null_count(arr: pa.Array, ctx) -> DeviceArray:
    """the same device buffers through from_pointers with null_count = -1 (how the hash join passes its build ids)"""
    d = dev(arr, ctx)
    return DeviceArray.from_pointers(ctx, arr.type, len(arr), d.buffers[1].ptr, validity_ptr=d.buffers[0].ptr,
                                     null_count=-1, offset=d.offset, keepalive=d)


# ---------------------------------------------------------------------------------------------------------------------
# sort_indices: values, sizes, offsets
# ---------------------------------------------------------------------------------------------------------------------
# (n, nv): both counts at k * tile +- 1, a last one-sweep tile with fewer keys than one warp's segment, nv = 0 and 1
SHAPES = [(0, 0), (1, 0), (1, 1), (2, 1), (TILE - 1, TILE - 1), (TILE + 1, TILE + 1), (TILE + 1, TILE - 1),
          (2 * PREP_TILE - 1, TILE + 1), (3 * PREP_TILE + 1, 3 * TILE - 1), (3 * TILE + 100, 3 * TILE + 100),
          (4 * PREP_TILE + 7, 2 * TILE + WARP_KEYS - 1), (5 * TILE + 1, 5 * TILE + 1), (6 * PREP_TILE - 1, 37)]
LARGE_N = 3_100_001          # ~3 M valid keys: ~740 one-sweep tiles, about two waves of 3 CTAs on each of 132 SMs


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_sort_indices_edges(ctx, t):
    rng = np.random.default_rng(SEED + sr.NUMERIC.index(t))
    for s, (n, nv) in enumerate(SHAPES):
        offset = s % 5                                  # validity bits at non-byte offsets
        m = n + offset
        valid = np.concatenate([rng.random(offset) < 0.5, exact_nulls(n, nv, rng)])
        arr = sr.to_arrow(t, sr.edge_values(t, m, rng), valid, offset)
        assert len(arr) == n and n - arr.null_count == nv
        d = dev(arr, ctx) if s % 2 == 0 or nv == n else unknown_null_count(arr, ctx)
        for order in sr.ORDERS:
            for placement in sr.PLACEMENTS:
                got = indices(bc.array_sort_indices(d, order, placement))
                assert_sorted_like(got, reference(arr, order, placement), f"{t} n={n} nv={nv} off={offset} {order} {placement}")
    arr = sr.edge_array(t, LARGE_N, rng, null_p=0.03, offset=3)
    d = unknown_null_count(arr, ctx)
    for order in sr.ORDERS:
        for placement in sr.PLACEMENTS:
            got = indices(bc.array_sort_indices(d, order, placement))
            assert_sorted_like(got, sr.sort_indices_np(arr, order, placement), f"{t} n={LARGE_N} {order} {placement}")


# ---------------------------------------------------------------------------------------------------------------------
# skipped radix passes
# ---------------------------------------------------------------------------------------------------------------------
def varying_bytes(arr: pa.Array) -> set:
    """the bytes of the valid values' bits that are not constant.  For integers the kernel's key is the value's bits XOR
    a constant (the sign flip) or NOT-ed, so these are exactly the digits whose radix pass runs."""
    b = er.bits(arr)[er.valid_mask(arr)]
    w = b.dtype.itemsize
    return {k for k in range(w) if len(np.unique((b >> b.dtype.type(8 * k)) & b.dtype.type(0xFF))) > 1}


def pass_skip_cases(rng, n):
    """(name, array, the bytes that must vary)"""
    def wrap(t, v, valid=None):
        return sr.to_arrow(t, v, rng.random(n + 3) > 0.1 if valid is None else valid, 3)
    m = n + 3
    u64 = lambda v: np.asarray(v, np.uint64)                                # noqa: E731
    yield "all_equal_int32", wrap(pa.int32(), np.full(m, 0x12345678, np.int32)), set()
    yield "all_equal_uint64_max", wrap(pa.uint64(), np.full(m, np.iinfo(np.uint64).max, np.uint64)), set()
    yield "all_equal_int8_min", wrap(pa.int8(), np.full(m, -128, np.int8)), set()
    for ft in (pa.float32(), pa.float64()):
        dt = sr.ew.np_dtype(ft)
        zeros = np.where(rng.random(m) < 0.5, dt.type(-0.0), dt.type(0.0)).astype(dt)
        yield f"signed_zeros_{ft}", wrap(ft, zeros), None
        u = er.UINT_OF_WIDTH[dt.itemsize]
        mant = rng.integers(1, 1 << (23 if dt.itemsize == 4 else 52), m, dtype=np.int64).astype(u)
        expo = u((0xFF << 23) if dt.itemsize == 4 else (0x7FF << 52))
        sign = np.where(rng.random(m) < 0.5, u(1) << u(8 * dt.itemsize - 1), u(0)).astype(u)
        yield f"nan_payloads_{ft}", wrap(ft, (mant | expo | sign).view(dt)), None
    for t in (pa.int64(), pa.uint64(), pa.int32()):
        w = t.bit_width // 8
        base = rng.integers(0, 1 << 64, dtype=np.uint64, endpoint=False)
        for k in sorted({0, 3, w - 1}):
            r = u64(rng.integers(0, 256, m)) << u64(8 * k)
            v = (base ^ r) & u64((1 << (8 * w)) - 1)
            yield f"one_digit_{t}_byte{k}", wrap(t, v.astype(er.UINT_OF_WIDTH[w]).view(sr.ew.np_dtype(t))), {k}
        if w == 8:
            v = base ^ u64(rng.integers(0, 256, m)) ^ (u64(rng.integers(0, 256, m)) << u64(56))
            yield f"bytes_0_and_7_{t}", wrap(t, v.view(sr.ew.np_dtype(t))), {0, 7}
    for t in (pa.int8(), pa.uint8(), pa.int16(), pa.uint16()):
        yield f"narrow_full_range_{t}", wrap(t, sr.full_range(t, m, rng)), set(range(t.bit_width // 8))
    # one valid row differs from all the others: each varying digit has one bin holding all keys but one
    for t, same, odd, varying in ((pa.int8(), 7, -7, {0}), (pa.uint16(), 0x1234, 0x4321, {0, 1}),
                                  (pa.int64(), 0x0102030405060708, 0x0102030445060708, {3})):
        v = np.full(m, same, sr.ew.np_dtype(t))
        valid = rng.random(m) > 0.1
        row = int(rng.integers(3, m))
        v[row], valid[row] = odd, True
        yield f"one_odd_row_{t}", wrap(t, v, valid), varying


def test_pass_skip_patterns(ctx):
    rng = np.random.default_rng(SEED + 20)
    n = 3 * TILE + 777
    for name, arr, want_varying in pass_skip_cases(rng, n):
        v = er.raw(arr)[er.valid_mask(arr)]
        if want_varying is None:                   # floats: every valid row in one class of the total order
            assert (v == 0).all() or np.isnan(v).all(), name
            assert len(np.unique(er.bits(v))) > 1, name     # ... with different bits: -0.0 and +0.0, or NaN payloads
        else:
            assert varying_bytes(arr) == want_varying, name
        d = dev(arr, ctx)
        for order in sr.ORDERS:
            for placement in sr.PLACEMENTS:
                got = indices(bc.array_sort_indices(d, order, placement))
                want = reference(arr, order, placement)
                if not want_varying:
                    ok = er.valid_mask(arr)
                    rows = np.flatnonzero(ok)
                    nulls = np.flatnonzero(~ok)
                    assert want.tolist() == (rows.tolist() + nulls.tolist() if placement == "at_end"
                                             else nulls.tolist() + rows.tolist()), name   # row order comes out
                assert_sorted_like(got, want, f"{name} {order} {placement}")


# ---------------------------------------------------------------------------------------------------------------------
# sort_payload
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [pa.int64(), pa.float32(), pa.uint8(), pa.float64()], ids=str)
def test_sort_payload_full_range(ctx, t):
    rng = np.random.default_rng(SEED + 30 + sr.NUMERIC.index(t))
    for n in (1, TILE - 1, 3 * TILE + 5, 200_001):
        arr = sr.edge_array(t, n, rng, null_p=0.1, offset=2)
        p = rng.integers(0, 1 << 32, n + 7, dtype=np.uint64).astype(np.uint32)
        p[rng.random(n + 7) < 0.2] = 0xFFFFFFFF
        pay = sr.to_arrow(pa.uint32(), p, None, 7)
        d, dp = dev(arr, ctx), dev(pay, ctx)
        for order in sr.ORDERS:
            for placement in sr.PLACEMENTS:
                got = bc.sort_payload(d, dp, order, placement).to_arrow()
                assert got.type == pa.uint64() and got.null_count == 0
                want = p[7:][reference(arr, order, placement)].astype(np.uint64)
                assert np.array_equal(got.to_numpy(), want), f"{t} n={n} {order} {placement}"


def test_sort_payload_errors(ctx):
    text = "b2_sort_payload: payload must be a uint32 array without nulls of the values' length"
    d = dev(pa.array(np.arange(10, dtype=np.int64)), ctx)
    bad = [pa.array(np.arange(10, dtype=np.int32)),                               # wrong type
           pa.array(np.arange(10, dtype=np.uint32), mask=np.arange(10) == 4),     # nulls
           pa.array(np.arange(9, dtype=np.uint32))]                               # length
    for p in bad:
        with pytest.raises(pa.ArrowInvalid, match=re.escape(text)):
            bc.sort_payload(d, dev(p, ctx))


# ---------------------------------------------------------------------------------------------------------------------
# multi-key sort
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("placement", sr.PLACEMENTS)
def test_multi_key_sort_edges(ctx, placement):
    """full-range and edge keys (ties on +-0 and on NaN payloads that must fall through to the next key), a utf8 key, and
    a different slice offset per column"""
    rng = np.random.default_rng(SEED + 40)
    for n in (1, 37, TILE + 1, 3 * TILE - 1, 20000):
        cols = sr.multi_columns(n, rng)
        dcols = {k: dev(v, ctx) for k, v in cols.items()}
        for keys in sr.MULTI_KEYS:
            names = [k for k, _ in keys]
            want = sr.sort_indices_multi_ref([cols[k] for k in names], [o for _, o in keys], placement)
            got = indices(bc.sort_indices({k: dcols[k] for k in names}, sort_keys=keys, null_placement=placement))
            assert_sorted_like(got, np.array(want, np.int64), f"n={n} {keys} {placement}")


def test_multi_key_sort_large(ctx):
    rng = np.random.default_rng(SEED + 41)
    n = 2_000_003
    cols = sr.multi_columns(n, rng)
    cols["l"] = sr.edge_array(pa.int64(), n, rng, null_p=0.01, offset=4)
    del cols["s"]
    dcols = {k: dev(v, ctx) for k, v in cols.items()}
    for keys in ([("f", "ascending"), ("u", "descending"), ("l", "ascending")],
                 [("g", "descending"), ("i", "ascending"), ("f", "descending"), ("u", "ascending")]):
        names = [k for k, _ in keys]
        for placement in sr.PLACEMENTS:
            want = sr.sort_indices_multi_np([cols[k] for k in names], [o for _, o in keys], placement)
            got = indices(bc.sort_indices({k: dcols[k] for k in names}, sort_keys=keys, null_placement=placement))
            assert_sorted_like(got, want, f"{keys} {placement}")


# ---------------------------------------------------------------------------------------------------------------------
# select_k
# ---------------------------------------------------------------------------------------------------------------------
def select_k_branch(arr: pa.Array, k: int, order: str, placement: str):
    """(branch, threshold) that b2_select_k takes on this input, restated from select_k.cu"""
    n = len(arr)
    k = min(k, n)
    is_float = pa.types.is_floating(arr.type)
    if k == 0:
        return "empty", None
    if n < SELECT_MIN_N:
        return "small_n", None
    if k * SELECT_K_FACTOR > n:
        return "large_k", None
    if placement == "at_start" and ((arr.null_count != 0 and arr.buffers()[0] is not None) or is_float):
        return "at_start", None
    stride = n // SAMPLE
    sample = arr.take(pa.array(np.arange(SAMPLE, dtype=np.int64) * stride + (stride >> 1)))
    perm = sr.sort_indices_np(sample, order, "at_end")
    rank = int(k / n * SAMPLE * 2.0) + 96
    if rank >= SAMPLE - 1:
        return "rank", None
    i = perm[rank]
    if not er.valid_mask(sample)[i]:
        return "sample_null", None
    t = er.raw(sample)[i]
    if is_float and np.isnan(t):
        return "nan_threshold", t
    v, valid = er.raw(arr), er.valid_mask(arr)
    with np.errstate(invalid="ignore"):
        m = int((valid & ((v <= t) if order == "ascending" else (v >= t))).sum())
    if m < k:
        return "few_candidates", t
    if m * 2 > n:
        return "many_candidates", t
    return "threshold", t


def check_select_k(ctx, arr, k, order, placement, branch, msg):
    got_branch, t = select_k_branch(arr, k, order, placement)
    assert got_branch == branch, f"{msg}: the data reaches {got_branch}, not {branch}"
    got = indices(bc.select_k_unstable(dev(arr, ctx), k, [("x", order)], null_placement=placement))
    assert_sorted_like(got, sr.sort_indices_np(arr, order, placement)[:k], msg)
    return t


def test_select_k_rank_fallback_is_a_guard_only():
    """the k switch (k * 8 <= n) keeps the sample rank at most SAMPLE / 4 + 96: the `rank >= kSample - 1` fallback cannot
    be reached while the switches stay as they are"""
    n = SELECT_MIN_N
    k = n // SELECT_K_FACTOR
    assert int(k / n * SAMPLE * 2.0) + 96 < SAMPLE - 1


def test_select_k_branches(ctx):
    rng = np.random.default_rng(SEED + 50)
    N = SELECT_MIN_N
    i64 = pa.int64()
    full = lambda t, n, null_p=0.0, off=0: sr.to_arrow(t, sr.full_range(t, n + off, rng), rng.random(n + off) >= null_p, off)  # noqa: E731
    # the size switch and the k switch, on both sides
    check_select_k(ctx, full(i64, N - 1), 10, "ascending", "at_end", "small_n", "n = 2^20 - 1")
    check_select_k(ctx, full(i64, N), 10, "ascending", "at_end", "threshold", "n = 2^20")
    a = full(i64, N, 0.05, 3)
    check_select_k(ctx, a, N // SELECT_K_FACTOR, "descending", "at_end", "threshold", "8k = n")
    check_select_k(ctx, a, N // SELECT_K_FACTOR + 1, "descending", "at_end", "large_k", "8k = n + 8")
    # the at_start guard: nulls possible, or floats (NaNs first would be skipped by the threshold)
    check_select_k(ctx, a, 100, "ascending", "at_start", "at_start", "int64 with nulls at_start")
    check_select_k(ctx, full(pa.float32(), N), 100, "ascending", "at_start", "at_start", "float32 at_start")
    check_select_k(ctx, full(pa.int32(), N, 0.0, 5), 100, "descending", "at_start", "threshold", "int32 no nulls at_start")
    # a NaN threshold: 95 % NaN, so the sample rank lands in the sample's NaNs
    v = sr.full_range(pa.float64(), N, rng)
    v[rng.random(N) < 0.95] = np.nan
    check_select_k(ctx, sr.to_arrow(pa.float64(), v), N // 20, "ascending", "at_end", "nan_threshold", "NaN threshold")
    # a null threshold: 95 % nulls
    check_select_k(ctx, full(pa.int32(), N, 0.95), N // 20, "descending", "at_end", "sample_null", "null threshold")
    # fewer candidates than k: the strided sample rows hold the least value, every other row a larger one
    stride = N // SAMPLE
    v = rng.integers(1, 1 << 40, N)
    v[np.arange(SAMPLE) * stride + (stride >> 1)] = 0
    check_select_k(ctx, sr.to_arrow(i64, v), 100_000, "ascending", "at_end", "few_candidates", "m < k")
    # more than half the rows at or before the threshold
    v = rng.integers(-1000, 1000, N)
    v[rng.random(N) < 0.6] = -5000
    check_select_k(ctx, sr.to_arrow(i64, v), 10, "ascending", "at_end", "many_candidates", "m * 2 > n")


def test_select_k_threshold_edges(ctx):
    rng = np.random.default_rng(SEED + 51)
    N = SELECT_MIN_N
    # ties across position k
    v = rng.integers(-3000, 3000, N + 12348).astype(np.int32)
    a = sr.to_arrow(pa.int32(), v, rng.random(N + 12348) > 0.05, 3)
    for order in sr.ORDERS:
        for k in (1000, 4097):
            check_select_k(ctx, a, k, order, "at_end", "threshold", f"ties {order} k={k}")
    # uint64 thresholds at or above 2^63
    lo = rng.integers(0, 1 << 20, N + 1).astype(np.uint64)
    for order, v in (("ascending", np.uint64(1 << 63) + lo), ("descending", np.uint64((1 << 64) - 1) - lo)):
        t = check_select_k(ctx, sr.to_arrow(pa.uint64(), v, rng.random(N + 1) > 0.02), 5000, order, "at_end", "threshold",
                           f"uint64 {order}")
        assert int(t) >= 1 << 63
    # INT64_MIN / INT64_MAX thresholds: a fifth of the rows hold the extreme
    for order, extreme in (("ascending", -(1 << 63)), ("descending", (1 << 63) - 1)):
        v = sr.full_range(pa.int64(), N + 2, rng)
        v[rng.random(N + 2) < 0.2] = extreme
        t = check_select_k(ctx, sr.to_arrow(pa.int64(), v, rng.random(N + 2) > 0.01, 2), 5000, order, "at_end", "threshold",
                           f"int64 {order} extreme")
        assert int(t) == extreme
    # a zero threshold of one sign with zeros of the other sign among the rows: all of them are candidates, and k reaches
    # past the rows before the zeros, so the first k rows hold zeros of both signs that must tie (row order)
    n = 2 * N
    stride = n // SAMPLE
    sample_rows = np.arange(SAMPLE) * stride + (stride >> 1)
    for t_, order, before, sample_zero in ((pa.float64(), "ascending", -1.0, -0.0), (pa.float32(), "descending", 1.0, 0.0)):
        dt = sr.ew.np_dtype(t_)
        mag = np.abs(sr.full_range(t_, n, rng))
        u = rng.random(n)
        with np.errstate(invalid="ignore"):
            v = np.where(u < 0.01, before * mag, -before * mag).astype(dt)   # 1 % before the zeros in the order, the rest after
        zero = (u >= 0.01) & (u < 0.31)
        v[zero] = np.where(rng.random(n) < 0.5, dt.type(-0.0), dt.type(0.0))[zero]
        on_sample = np.zeros(n, bool)
        on_sample[sample_rows] = True
        v[zero & on_sample] = dt.type(sample_zero)                         # the threshold is a zero of this sign ...
        a = sr.to_arrow(t_, v, rng.random(n) > 0.02)
        k = 40000
        t = check_select_k(ctx, a, k, order, "at_end", "threshold", f"{t_} zero threshold {order}")
        assert t == 0 and np.signbit(t) == np.signbit(sample_zero)
        prefix = sr.sort_indices_np(a, order, "at_end")[:k]
        zero_rows = prefix[v[prefix] == 0]                                   # ... and the first k hold zeros of both signs,
        signs = np.signbit(v[zero_rows])                                     # interleaved in row order
        assert 1000 < len(zero_rows) < k and np.all(np.diff(zero_rows) > 0)
        assert signs.any() and (~signs).any() and np.count_nonzero(signs[1:] != signs[:-1]) > 100
    # full-range floats, sliced: few edge values, so the threshold and most of the first k rows are finite
    for t_ in (pa.float32(), pa.float64()):
        a = sr.edge_array(t_, N + 1, rng, null_p=0.05, offset=5, edge_p=0.01)
        v = er.raw(a)
        for order in sr.ORDERS:
            k = 3000
            t = check_select_k(ctx, a, k, order, "at_end", "threshold", f"{t_} full range {order}")
            assert np.isfinite(t)
            assert np.count_nonzero(np.isfinite(v[sr.sort_indices_np(a, order, "at_end")[:k]])) > k // 2


# ---------------------------------------------------------------------------------------------------------------------
# range_partition / range_split and the distributed sort's composition
# ---------------------------------------------------------------------------------------------------------------------
def range_partition(ctx, d, ds, order) -> np.ndarray:
    cv, cs, out = d._c(), ds._c(), cabi.B2Array()
    check(ctx.lib.b2_range_partition(ctx.handle, C.byref(cv), C.byref(cs), ORDER_ID[order], C.byref(out), ctx.stream))
    return DeviceArray._from_c(ctx, out, pa.uint32()).to_arrow().to_numpy().astype(np.int64)


def range_split(ctx, d, ds, order, row_base):
    n_bins = ds.length + 2
    counts = (C.c_int64 * n_bins)()
    cv, cs, ov, orows = d._c(), ds._c(), cabi.B2Array(), cabi.B2Array()
    check(ctx.lib.b2_range_split(ctx.handle, C.byref(cv), C.byref(cs), ORDER_ID[order], row_base, C.byref(ov), C.byref(orows),
                                 counts, ctx.stream))
    return DeviceArray._from_c(ctx, ov, d.type), DeviceArray._from_c(ctx, orows, pa.uint32()), list(counts)


def splitter_sets(t, rng, most):
    pool = sr.edge_pool(t)
    yield "none", pool[:0]
    yield "one", pool[len(pool) // 2:len(pool) // 2 + 1]
    yield "max", pool[rng.integers(0, len(pool), most)]              # duplicates, +-0, NaNs, +-inf, integer extremes


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_range_partition_and_split(ctx, t):
    rng = np.random.default_rng(SEED + 60 + sr.NUMERIC.index(t))
    n = 5 * 2048 + 17
    arr = sr.edge_array(t, n, rng, null_p=0.1, offset=3, edge_p=0.6)
    d = dev(arr, ctx)
    raw_bits = er.bits(arr)
    for order in sr.ORDERS:
        for name, most in (("partition", PARTITION_MAX), ("split", SPLIT_MAX)):
            for label, sp in splitter_sets(t, rng, most):
                msg = f"{t} {order} {name} {label}"
                ds = dev(sr.to_arrow(t, sp), ctx)
                want = sr.range_bins_np(arr, sp.tolist(), order)
                if name == "partition":
                    assert_sorted_like(range_partition(ctx, d, ds, order), want, msg)
                    continue
                row_base = 1000 if label != "max" else (1 << 32) - 1 - n         # the largest row_base accepted
                vals, rows, counts = range_split(ctx, d, ds, order, row_base)
                assert counts == np.bincount(want, minlength=len(sp) + 2).tolist(), msg
                perm = np.argsort(want, kind="stable")
                assert_sorted_like(rows.to_arrow().to_numpy().astype(np.int64), perm + row_base, msg)
                assert vals.to_arrow().null_count == 0
                assert np.array_equal(er.bits(vals.to_arrow()), raw_bits[perm]), msg
        for name, most, fn in (("partition", PARTITION_MAX, lambda ds: range_partition(ctx, d, ds, order)),
                               ("split", SPLIT_MAX, lambda ds: range_split(ctx, d, ds, order, 0))):
            ds = dev(sr.to_arrow(t, sr.edge_pool(t)[rng.integers(0, len(sr.edge_pool(t)), most + 1)]), ctx)
            with pytest.raises(pa.ArrowInvalid, match=f"at most {most} splitters"):
                fn(ds)
    with pytest.raises(pa.ArrowNotImplementedError, match="row numbers must fit 32 bits"):
        range_split(ctx, d, dev(sr.to_arrow(t, sr.edge_pool(t)[:1]), ctx), "ascending", (1 << 32) - n)


@pytest.mark.parametrize("t", sr.NUMERIC, ids=str)
def test_range_split_then_sort_payload_is_the_global_sort(ctx, t):
    """the distributed sort's argument on one device: bins in splitter order, each bin sorted with its row numbers as the
    payload, then the null bin, give array_sort_indices(values, order, "at_end")"""
    rng = np.random.default_rng(SEED + 70 + sr.NUMERIC.index(t))
    n = 7 * 2048 + 3
    arr = sr.edge_array(t, n, rng, null_p=0.1, offset=1, edge_p=0.6)
    d = dev(arr, ctx)
    pool = sr.edge_pool(t)
    for order in sr.ORDERS:
        for count in (0, 1, 7, SPLIT_MAX):
            sp = sorted(pool[rng.integers(0, len(pool), count)].tolist(), key=lambda s: sr.range_key(s, order))
            ds = dev(sr.to_arrow(t, np.array(sp, dtype=sr.ew.np_dtype(t))), ctx)
            vals, rows, counts = range_split(ctx, d, ds, order, 0)
            out, start = [], 0
            for b, c in enumerate(counts):
                if b < len(counts) - 1 and c:
                    out.append(indices(bc.sort_payload(vals.slice(start, c), rows.slice(start, c), order, "at_end")))
                elif c:
                    out.append(rows.slice(start, c).to_arrow().to_numpy().astype(np.int64))
                start += c
            got = np.concatenate(out) if out else np.zeros(0, np.int64)
            assert_sorted_like(got, reference(arr, order, "at_end"), f"{t} {order} {count} splitters")
            assert_sorted_like(got, indices(bc.array_sort_indices(d, order, "at_end")), f"{t} {order} {count} splitters")


# ---------------------------------------------------------------------------------------------------------------------
# the 2^30 boundary of the look-back cells, and the 2^32 refusal
# ---------------------------------------------------------------------------------------------------------------------
FULLSIZE = int(os.environ.get("B200_FULLSIZE_ROWS", "1000000000"))


@pytest.fixture()
def big_torch(ctx):
    """these sorts and their device-side checks need about 25-30 GB of device memory"""
    import gc

    import torch
    if FULLSIZE < 1_000_000_000:
        pytest.skip("full-size run only (B200_FULLSIZE_ROWS)")
    gc.collect()
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()
    free, _ = torch.cuda.mem_get_info()
    if free < 36 << 30:
        pytest.skip(f"needs ~36 GiB of free device memory, {free >> 30} GiB free")
    return torch


def check_on_device(ctx, torch, keys_t, order):
    """a permutation, keys in order, and row numbers increasing within ties -- on the device, nothing crosses PCIe"""
    from tests.test_gpu_fullsize import as_tensor
    n = keys_t.numel()
    dtype = {torch.int8: pa.int8(), torch.int16: pa.int16()}[keys_t.dtype]
    keys = DeviceArray.from_pointers(ctx, dtype, n, keys_t.data_ptr())
    torch.cuda.synchronize()
    out = bc.array_sort_indices(keys, order)
    ctx.sync()
    ctx.trim()
    idx = as_tensor(torch, out, torch.int64)
    seen = torch.zeros(n, dtype=torch.bool, device="cuda")
    seen[idx] = True
    assert bool(seen.all())
    del seen
    sk = keys_t[idx]
    step = sk[1:].to(torch.int16) - sk[:-1].to(torch.int16)
    assert bool((step >= 0).all()) if order == "ascending" else bool((step <= 0).all())
    bad = (step == 0) & (idx[1:] <= idx[:-1])
    assert not bool(bad.any())                            # stable
    return idx


@pytest.mark.parametrize("n", [(1 << 30) - 1, 1 << 30], ids=["2^30-1", "2^30"])
def test_fullsize_one_bin_holds_all_but_one_row(ctx, big_torch, n):
    """int8 keys, all 0 but one 1: a single radix pass whose bin 0 holds n - 1 keys -- the largest count the 30-bit look-back
    cells carry (n = 2^30 - 1) and the first size with 64-bit cells (n = 2^30)"""
    torch = big_torch
    keys_t = torch.zeros(n, dtype=torch.int8, device="cuda")
    odd = n // 3
    keys_t[odd] = 1
    for order in sr.ORDERS:
        idx = check_on_device(ctx, torch, keys_t, order)
        assert int(idx[-1 if order == "ascending" else 0].item()) == odd
        del idx


def test_fullsize_stable_beyond_2_30(ctx, big_torch):
    """2^30 + 70001 int16 keys with ~10^6 rows per value: stability on the 64-bit look-back path is actually exercised"""
    torch = big_torch
    n = (1 << 30) + 70001
    gen = torch.Generator(device="cuda").manual_seed(SEED + 80)
    keys_t = torch.randint(-500, 500, (n,), dtype=torch.int16, device="cuda", generator=gen)
    for order in sr.ORDERS:
        check_on_device(ctx, torch, keys_t, order)


def test_sort_refuses_2_32_rows_before_touching_memory(ctx):
    """arrays of SORT_LIMIT rows or more are refused before anything is allocated or launched: the views below claim that
    many rows over a 64-byte buffer"""
    tiny = dev(pa.array(np.zeros(16, np.uint32)), ctx)
    big = {t: DeviceArray.from_pointers(ctx, t, SORT_LIMIT, tiny.buffers[1].ptr, keepalive=tiny) for t in (pa.int32(), pa.uint32())}
    text = "arrays of 2^32 rows or more must be sorted as chunks"
    with pytest.raises(pa.ArrowNotImplementedError, match=re.escape(text)):
        bc.array_sort_indices(big[pa.int32()])
    with pytest.raises(pa.ArrowNotImplementedError, match=re.escape(text)):
        bc.sort_payload(big[pa.int32()], big[pa.uint32()])
    with pytest.raises(pa.ArrowNotImplementedError, match=re.escape(text)):
        bc.sort_indices({"a": big[pa.int32()], "b": big[pa.uint32()]}, sort_keys=[("a", "ascending"), ("b", "descending")])
