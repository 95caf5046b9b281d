"""Sorting by utf8 / binary keys on the device (csrc/sort_strings.cu: a uint32 rank per row, then the numeric radix
sort): array_sort_indices, sort_indices over tables with string and numeric keys, sort_payload and select_k_unstable,
each against the restated sort (tests/string_sort_oracle.py) and the reference binary.  The long-shared-prefix inputs bound the refinement rounds: they
must finish in seconds, not in one round per 7 bytes."""
import time

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import string_sort_oracle as sso
from tests.sort_string_cases import (STRING_TYPES, cases, random_bytes, shared_prefix_strings, strings_array,
                                     two_long_identical)
from tests.util import SEED, assert_equal, random_array

pytestmark = pytest.mark.gpu
ORDERS = ["ascending", "descending"]
PLACEMENTS = ["at_end", "at_start"]


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


def check_sort(ctx, arr, msg):
    d = dev(arr, ctx)
    for order in ORDERS:
        for placement in PLACEMENTS:
            got = bc.array_sort_indices(d, order, placement).to_arrow()
            assert_equal(got, sso.sort_indices(arr, order, placement), f"{msg} {order} {placement} (oracle)")
            assert_equal(got, pc.array_sort_indices(arr, order=order, null_placement=placement), f"{msg} {order} {placement}")


@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_string_sort_cases(ctx, t):
    for name, vals, null_p in cases():
        for offset in (0, 3):
            check_sort(ctx, strings_array(t, vals, null_p, SEED, offset=offset), f"{t} {name} offset={offset}")


@pytest.mark.parametrize("t", [pa.string(), pa.large_binary()], ids=str)
def test_string_sort_300k(ctx, t):
    arr = strings_array(t, random_bytes(300_000, SEED + 11, max_len=40), 0.1, SEED, offset=1)
    check_sort(ctx, arr, f"{t} n=300000")


@pytest.mark.parametrize("shift", [1, 3])
def test_string_sort_odd_address(ctx, shift):
    """a character buffer that starts at an odd device address"""
    t = pa.large_binary()
    vals = strings_array(t, random_bytes(20000, SEED + shift), 0.1, SEED)
    aligned = dev(vals, ctx)
    data = np.ascontiguousarray(np.frombuffer(vals.buffers()[2], dtype=np.uint8))
    raw = ctx.alloc(len(data) + 16)
    ctx.h2d(raw.ptr + shift, data.ctypes.data, len(data))
    ctx.sync()
    moved = DeviceArray.from_pointers(ctx, t, len(vals), aligned.buffers[1].ptr, validity_ptr=aligned.buffers[0].ptr,
                                      null_count=vals.null_count, data2_ptr=raw.ptr + shift, keepalive=(aligned, raw))
    for order in ORDERS:
        got = bc.array_sort_indices(moved, order).to_arrow()
        assert_equal(got, pc.array_sort_indices(vals, order=order), f"shift={shift} {order}")


@pytest.mark.parametrize("name", ["shared 64 KiB prefix", "two identical 1 MiB strings"])
def test_string_sort_round_bound(ctx, name):
    vals = shared_prefix_strings(SEED) if name.startswith("shared") else two_long_identical(SEED)
    arr = strings_array(pa.large_binary(), vals, 0.05, SEED, offset=2)
    d = dev(arr, ctx)
    bc.array_sort_indices(d).to_arrow()  # module load
    t0 = time.perf_counter()
    for order in ORDERS:
        for placement in PLACEMENTS:
            got = bc.array_sort_indices(d, order, placement).to_arrow()
            assert_equal(got, pc.array_sort_indices(arr, order=order, null_placement=placement), f"{name} {order} {placement}")
    assert time.perf_counter() - t0 < 20.0, f"{name}: the refinement rounds grow with the string length"


def test_sort_payload_strings(ctx):
    arr = strings_array(pa.string(), random_bytes(50_000, SEED + 5, max_len=12, alphabet=b"abc\x00\xff"), 0.1, SEED, offset=5)
    payload = pa.array(np.random.default_rng(SEED).integers(0, 2**32 - 1, len(arr), dtype=np.uint32))
    for order in ORDERS:
        for placement in PLACEMENTS:
            got = bc.sort_payload(dev(arr, ctx), dev(payload, ctx), order, placement).to_arrow()
            idx = sso.sort_indices(arr, order, placement)
            assert_equal(got, pc.take(payload, idx).cast(pa.uint64()), f"{order} {placement}")


def test_table_sort_string_and_numeric_keys(ctx):
    n = 60_000
    cols = {
        "s": strings_array(pa.string(), random_bytes(n, SEED, max_len=9, alphabet=b"xyz"), 0.1, SEED + 1, offset=3),
        "i": random_array(pa.int64(), n, 0.1, SEED + 2, lo=-3, hi=3, offset=1),
        "b": strings_array(pa.large_binary(), random_bytes(n, SEED + 3, max_len=2, alphabet=b"\x00\xff"), 0.05, SEED + 4),
        "f": random_array(pa.float32(), n, 0.0, SEED + 5, lo=0, hi=4),
    }
    dcols = {k: dev(v, ctx) for k, v in cols.items()}
    for keys in ([("s", "descending"), ("i", "ascending")], [("i", "descending"), ("b", "ascending"), ("s", "ascending")],
                 [("b", "descending"), ("s", "descending"), ("f", "ascending")], [("s", "ascending")]):
        for placement in PLACEMENTS:
            got = bc.sort_indices(dcols, keys, placement).to_arrow()
            assert_equal(got, sso.sort_indices_multi(cols, keys, placement), f"{keys} {placement} (oracle)")
            assert_equal(got, pc.sort_indices(pa.table(cols), sort_keys=keys, null_placement=placement), f"{keys} {placement}")


@pytest.mark.parametrize("t", [pa.string(), pa.large_binary()], ids=str)
def test_select_k_strings(ctx, t):
    s = dev(pa.array(["b", "a", None, "a"], pa.string()).cast(t), ctx)
    assert bc.select_k_unstable(s, 3, [("x", "descending")]).to_arrow().to_pylist() == [0, 1, 3]
    # 2M rows take the sampled-threshold path for small k, the full sort for large k
    for n, null_p in ((2_000_000, 0.1), (5000, 0.0)):
        arr = strings_array(t, random_bytes(n, SEED + n, max_len=10, alphabet=b"abcdefgh"), null_p, SEED, offset=1)
        d = dev(arr, ctx)
        for order in ORDERS:
            full = bc.array_sort_indices(d, order).to_arrow()
            assert_equal(full, pc.array_sort_indices(arr, order=order), f"{t} n={n} {order}")
            if n <= 5000:
                assert_equal(full, sso.sort_indices(arr, order), f"{t} n={n} {order}")
            for k in (0, 1, 100, 5000, n + 3):
                got = bc.select_k_unstable(d, k, [("x", order)]).to_arrow()
                assert got.equals(full.slice(0, min(k, n))), f"{t} n={n} {order} k={k}"
            want = pc.select_k_unstable(arr, 1000, [("x", order)])
            got = bc.select_k_unstable(d, 1000, [("x", order)]).to_arrow()
            assert pc.take(arr, got).equals(pc.take(arr, want)), f"{t} n={n} {order}"
