"""is_in / index_in on the device (csrc/set_lookup.cu) against pyarrow.compute and the exact restatement
(set_lookup_ref), null slots included: every type x every null-matching behaviour x both functions, lengths around the
32-row warp groups, offsets on both sides, value sets on both sides of the shared / global table threshold, keys built to
collide, long strings, implicit casts, errors, lists of chunks and an input of more than 2^30 rows."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi
from tests import hash_keys as hk
from tests import set_lookup_ref as ref
from tests.test_set_lookup_oracle import STRINGS, TYPES, random_pair

pytestmark = pytest.mark.gpu
BEHAVIORS = ref.BEHAVIORS
FUNCTIONS = ("is_in", "index_in")


def _raw_data(arr: pa.Array, function: str) -> np.ndarray:
    """the result's data, slots under nulls included"""
    if function == "index_in":
        return np.frombuffer(arr.buffers()[1], np.int32, count=arr.offset + len(arr))[arr.offset:]
    bits = np.unpackbits(np.frombuffer(arr.buffers()[1], np.uint8), bitorder="little")
    return bits[arr.offset:arr.offset + len(arr)].astype(bool)


def check(ctx, values: pa.Array, value_set, behavior: str, function: str):
    dv = DeviceArray.from_arrow(values, ctx)
    dvs = value_set if isinstance(value_set, DeviceArray) else DeviceArray.from_arrow(value_set, ctx)
    got = getattr(bc, function)(dv, dvs, null_matching_behavior=behavior).to_arrow()
    host_set = value_set.to_arrow() if isinstance(value_set, DeviceArray) else value_set
    data, valid = ref.set_lookup(values, host_set, behavior, function)
    want = ref.to_arrow(data, valid, function)
    assert got.equals(want), (function, behavior, values.type, len(values), len(host_set))
    np.testing.assert_array_equal(_raw_data(got, function), np.where(valid, data, 0).astype(data.dtype))
    if behavior in ("match", "skip"):
        assert got.equals(getattr(pc, function)(values, value_set=host_set, skip_nulls=behavior == "skip"))
    return got


@pytest.mark.parametrize("tname", list(TYPES))
@pytest.mark.parametrize("behavior", BEHAVIORS)
@pytest.mark.parametrize("function", FUNCTIONS)
def test_types_behaviours(ctx, tname, behavior, function):
    rng = np.random.default_rng(len(tname) * 131 + BEHAVIORS.index(behavior) * 7 + FUNCTIONS.index(function))
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 1000):
        for m in (0, 1, 8):
            vals, vs = random_pair(tname, rng, n + 5, m + 3)
            check(ctx, vals.slice(0, n), vs.slice(0, m), behavior, function)
            check(ctx, vals.slice(5), vs.slice(3), behavior, function)   # offsets on both sides, not byte-aligned
    check(ctx, vals, pa.array([None] * 4, TYPES[tname]), behavior, function)


def _int64_pair(rng, n, m, null_p=0.1):
    vs = rng.integers(-(1 << 40), 1 << 40, m, dtype=np.int64)
    pick = rng.integers(0, max(m, 1), n)
    hits = vs[pick] if m else np.zeros(n, np.int64)
    vals = np.where(rng.random(n) < 0.5, hits, rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64))
    return pa.array(vals, mask=rng.random(n) < null_p), pa.array(vs, mask=rng.random(m) < 0.001)


def shared_threshold(ctx) -> int:
    """the most distinct values whose table the probe stages in shared memory (a power of two: the table has 2x as many
    slots, rounded up to a power of two)"""
    t = 1
    while bc.set_lookup_table(DeviceArray.from_arrow(pa.array(np.arange(2 * t, dtype=np.int64)), ctx))[1]:
        t *= 2
    return t


def test_shared_threshold(ctx):
    """two 512-thread probe blocks still share an SM: on the H100 (228 KB per SM) that is 4096 distinct values"""
    t = shared_threshold(ctx)
    assert t == 4096
    assert bc.set_lookup_table(DeviceArray.from_arrow(pa.array(np.arange(t, dtype=np.int64)), ctx))[1]
    assert not bc.set_lookup_table(DeviceArray.from_arrow(pa.array(np.arange(t + 1, dtype=np.int64)), ctx))[1]


@pytest.mark.parametrize("m", [0, 1, 8, 4096, 4097, 8193, 1 << 20, 10_000_000])
def test_set_sizes_and_placement(ctx, m):
    """the table is staged in shared memory up to the threshold and probed in global memory above"""
    rng = np.random.default_rng(m)
    vals, vs = _int64_pair(rng, (1 << 20) + 77, m + 3)
    vs = vs.slice(3)
    nbytes, shared = bc.set_lookup_table(DeviceArray.from_arrow(vs, ctx))
    distinct = len(pc.unique(vs.drop_null()))
    assert shared == (distinct <= shared_threshold(ctx)), (m, distinct, nbytes)
    for behavior in ("match", "inconclusive"):
        for function in FUNCTIONS:
            check(ctx, vals.slice(77), vs, behavior, function)


def test_string_placement_and_long_values(ctx):
    rng = np.random.default_rng(3)
    prefix = "p" * 300
    words = [prefix + str(i) for i in range(9000)]
    vals = pa.array([words[i] if i % 3 else "x" + words[i] for i in rng.integers(0, 9000, 50_000)], pa.large_string())
    for m in (4096, 4097, 9000):
        vs = pa.array(words[:m], pa.large_string())
        assert bc.set_lookup_table(DeviceArray.from_arrow(vs, ctx))[1] == (m <= 4096)
        for function in FUNCTIONS:
            check(ctx, vals, vs, "match", function)
    big = "b" * (1 << 20)
    vals = pa.array([big, big[:-1] + "c", big[:-1], "", None, big], pa.string())
    for behavior in BEHAVIORS:
        for function in FUNCTIONS:
            check(ctx, vals, pa.array(["", big, None], pa.string()), behavior, function)
            check(ctx, vals.cast(pa.large_binary()), pa.array([b"", big.encode()], pa.large_binary()), behavior, function)


def test_colliding_keys(ctx):
    """keys whose hash64 share the low bits of a 1024-slot table: one probe chain 500 long, in shared and global memory"""
    keys = hk.keys_with_fields(500, hk.slot_field(10), seed=5)
    rng = np.random.default_rng(11)
    vals = pa.array(np.concatenate([keys, keys + 1, rng.choice(keys, 5000)]), mask=rng.random(6000) < 0.05)
    for function in FUNCTIONS:
        for behavior in BEHAVIORS:
            check(ctx, vals, pa.array(keys[::-1]), behavior, function)
    many = np.concatenate([keys, hk.filler_keys(20000, [], seed=9, exclude=keys)])
    assert not bc.set_lookup_table(DeviceArray.from_arrow(pa.array(many), ctx))[1]
    check(ctx, vals, pa.array(many), "match", "index_in")


def test_special_values(ctx):
    """-0.0 / +0.0, NaN payloads, all-ones bit patterns (the table's empty marker), extremes"""
    nan2 = np.frombuffer(np.uint64(0x7ff8000000000001).tobytes(), np.float64)[0]
    ones = np.frombuffer(np.uint64(0xffffffffffffffff).tobytes(), np.float64)[0]
    vals = pa.array(np.array([0.0, -0.0, np.nan, nan2, ones, np.inf], np.float64))
    for vs in ([-0.0, nan2], [ones, 0.0], [np.nan]):
        for function in FUNCTIONS:
            check(ctx, vals, pa.array(np.array(vs, np.float64)), "match", function)
    ivals = pa.array([-1, 0, 1, -1, np.iinfo(np.int64).min, np.iinfo(np.int64).max], pa.int64())
    for function in FUNCTIONS:
        check(ctx, ivals, pa.array([5, -1, -1, np.iinfo(np.int64).max], pa.int64()), "skip", function)
        check(ctx, ivals.cast(pa.uint64(), safe=False), pa.array([2**64 - 1, 0], pa.uint64()), "match", function)


def test_implicit_casts(ctx):
    i8 = DeviceArray.from_arrow(pa.array(range(9), pa.int8()), ctx)
    assert bc.is_in(i8, pa.array([2, 3, 5, 7], pa.int32())).to_arrow().to_pylist() == \
        [False, False, True, True, False, True, False, True, False]
    # [1.5, 2.0] cannot be cast to int32 safely: the input is cast to float64 instead
    i32 = pa.array([1, 2, None, 3, 2], pa.int32())
    got = bc.is_in(DeviceArray.from_arrow(i32, ctx), pa.array([1.5, 2.0]))
    assert got.to_arrow().equals(pc.is_in(i32, value_set=pa.array([1.5, 2.0])))
    got = bc.index_in(DeviceArray.from_arrow(i32, ctx), pa.array([1.5, 2.0]))
    assert got.to_arrow().equals(pc.index_in(i32, value_set=pa.array([1.5, 2.0])))
    # 2^40 does not fit int32: the int32 input is cast to int64
    big = pa.array([1 << 40, 3, 2], pa.int64())
    for fn in FUNCTIONS:
        got = getattr(bc, fn)(DeviceArray.from_arrow(i32, ctx), DeviceArray.from_arrow(big, ctx))
        assert got.to_arrow().equals(getattr(pc, fn)(i32, value_set=big))
    # a chunked value set: positions continue across the chunks
    chunked = pa.chunked_array([pa.array([7, 2], pa.int64()), pa.array([3, 2], pa.int64())])
    got = bc.index_in(DeviceArray.from_arrow(pa.array([2, 3, 4], pa.int64()), ctx), chunked)
    assert got.to_arrow().to_pylist() == [1, 2, None]


def test_errors(ctx):
    s = DeviceArray.from_arrow(pa.array(["aaa", None], pa.string()), ctx)
    d = DeviceArray.from_arrow(pa.array([1.0, 2.0]), ctx)
    with pytest.raises(pa.ArrowTypeError, match="Array type doesn't match type of values set"):
        bc.is_in(s, pa.array([1.0, 2.0]))
    with pytest.raises(pa.ArrowTypeError, match="Array type doesn't match type of values set"):
        bc.is_in(d, pa.array(["aaa"], pa.large_string()))
    with pytest.raises(pa.ArrowInvalid, match="without SetLookupOptions"):
        bc.call_function("is_in", [d])
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.is_in(s, pa.array(["aaa"], pa.large_string()))   # no device cast between string types
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.is_in(DeviceArray.from_arrow(pa.array([1, 2], pa.int32()).dictionary_encode(), ctx), pa.array([1], pa.int32()))
    assert bc.call_function("index_in", [d], {"value_set": pa.array([2.0]), "skip_nulls": True}).to_arrow().to_pylist() == [None, 0]
    lib, h = ctx.lib, C.c_void_p()
    # C-ABI codes: unsupported types, an over-long value set (refused before its buffers are read), a type mismatch
    for t in (_cabi.NA, _cabi.HALF_FLOAT, _cabi.FIXED_SIZE_BINARY):
        a = _cabi.B2Array(None, None, None, 0, 0, 0, t, 16)
        assert lib.b2_set_lookup_create(ctx.handle, C.byref(a), 0, C.byref(h), ctx.stream) == _cabi.NOT_IMPLEMENTED
    dummy = ctx.alloc(64)
    a = _cabi.B2Array(None, dummy.ptr, None, 1 << 31, 0, 0, _cabi.INT64, 0)
    assert lib.b2_set_lookup_create(ctx.handle, C.byref(a), 0, C.byref(h), ctx.stream) == _cabi.CAPACITY_ERROR
    cvs = d._c()
    assert lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), 4, C.byref(h), ctx.stream) == _cabi.INVALID
    assert lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), 0, C.byref(h), ctx.stream) == _cabi.OK
    try:
        wrong, out = DeviceArray.from_arrow(pa.array([1], pa.int64()), ctx)._c(), _cabi.B2Array()
        assert lib.b2_is_in(h, C.byref(wrong), C.byref(out), ctx.stream) == _cabi.TYPE_ERROR
        assert "doesn't match" in _cabi.last_error()
    finally:
        lib.b2_set_lookup_destroy(h)


def test_chunks_one_build(ctx):
    """a list of chunks: one table, one probe launch per chunk"""
    rng = np.random.default_rng(21)
    vals, vs = _int64_pair(rng, 300_000, 1000)
    chunks = [vals.slice(0, 1000), vals.slice(1000, 0), vals.slice(1001, 100_000), vals.slice(101_001)]
    dchunks = [DeviceArray.from_arrow(c, ctx) for c in chunks]
    dvs = DeviceArray.from_arrow(vs, ctx)
    lib = ctx.lib
    for fn in FUNCTIONS:
        before = lib.b2_launch_count()
        h = C.c_void_p()
        cvs = dvs._c()
        assert lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), 0, C.byref(h), ctx.stream) == 0
        try:
            for c, dc in zip(chunks, dchunks):
                start = lib.b2_launch_count()
                cc, co = dc._c(), _cabi.B2Array()
                assert getattr(lib, "b2_" + fn)(h, C.byref(cc), C.byref(co), ctx.stream) == 0
                assert lib.b2_launch_count() - start == (1 if len(c) else 0)
                got = bc._out(ctx, co, pa.int32() if fn == "index_in" else pa.bool_()).to_arrow()
                assert got.equals(getattr(pc, fn)(c, value_set=vs))
        finally:
            lib.b2_set_lookup_destroy(h)
        assert lib.b2_launch_count() > before
        outs = getattr(bc, fn)(dchunks, vs)
        assert len(outs) == len(chunks)
        for c, o in zip(chunks, outs):
            assert o.to_arrow().equals(getattr(pc, fn)(c, value_set=vs))


def test_more_than_2_30_rows(ctx):
    """2^30 + 4099 int8 rows against torch.isin: the count of true rows and of true bits is size-independent"""
    torch = pytest.importorskip("torch")
    n = (1 << 30) + 4099
    g = torch.Generator(device="cuda").manual_seed(5)
    t = torch.randint(-128, 128, (n,), dtype=torch.int8, device="cuda", generator=g)
    torch.cuda.synchronize()
    dv = DeviceArray.from_pointers(ctx, pa.int8(), n, t.data_ptr(), keepalive=t)
    setv = [-128, -3, 0, 5, 127]
    got = bc.is_in(dv, pa.array(setv, pa.int8()))
    assert len(got) == n and got.null_count == 0
    want = int(torch.isin(t, torch.tensor(setv, dtype=torch.int8, device="cuda")).sum())
    cnt = C.c_int64()
    cg = got._c()
    assert ctx.lib.b2_bitmap_count(ctx.handle, C.c_void_p(cg.data), 0, n, C.byref(cnt), ctx.stream) == 0
    assert cnt.value == want
    idx = bc.index_in(dv, pa.array(setv, pa.int8()))
    assert idx.null_count == n - want
    tail = idx.slice(n - 4099).to_arrow()
    tv = t[n - 4099:].cpu().numpy()
    assert tail.equals(pc.index_in(pa.array(tv), value_set=pa.array(setv, pa.int8())))
