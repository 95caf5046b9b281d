"""Every entry point that picks a kernel template from a type id or a byte width, called with every type id.

A rejected id must give the exact status code and message; an accepted id must return OK on a small input (the
exact-reference tests check the values).  Every array gets real device buffers, zero-filled and large enough for
16-byte values, so that an accepted call reads only in-bounds memory and every index is 0."""
import ctypes as C

import pytest

from arrow_b200 import _cabi as cb

pytestmark = pytest.mark.gpu

N = 4
ALL_IDS = list(range(16)) + [cb.LIST, cb.LARGE_STRING, cb.LARGE_BINARY]
NUMERIC = [cb.UINT8, cb.INT8, cb.UINT16, cb.INT16, cb.UINT32, cb.INT32, cb.UINT64, cb.INT64, cb.FLOAT, cb.DOUBLE]
INTEGER = NUMERIC[:8]
BINARY_LIKE = [cb.STRING, cb.BINARY, cb.LARGE_STRING, cb.LARGE_BINARY]
WIDTH = {cb.UINT8: 1, cb.INT8: 1, cb.UINT16: 2, cb.INT16: 2, cb.HALF_FLOAT: 2, cb.UINT32: 4, cb.INT32: 4, cb.FLOAT: 4,
         cb.UINT64: 8, cb.INT64: 8, cb.DOUBLE: 8}
NAMES = {cb.BOOL: "bool", cb.INT8: "int8", cb.UINT8: "uint8", cb.INT16: "int16", cb.UINT16: "uint16", cb.INT32: "int32",
         cb.UINT32: "uint32", cb.INT64: "int64", cb.UINT64: "uint64", cb.FLOAT: "float", cb.DOUBLE: "double",
         cb.STRING: "string", cb.BINARY: "binary", cb.LARGE_STRING: "large_string", cb.LARGE_BINARY: "large_binary"}
FSB_WIDTH = 16  # byte width of every fixed_size_binary array here


def sum_type(t):
    if t in (cb.FLOAT, cb.DOUBLE):
        return cb.DOUBLE
    return cb.INT64 if t in (cb.INT8, cb.INT16, cb.INT32, cb.INT64) else cb.UINT64


class Bufs:
    """Zeroed device buffers, freed at the end of the test, and the outputs of the calls."""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def zeros(self, nbytes):
        p = C.c_void_p()
        assert self.ctx.lib.b2_alloc(self.ctx.handle, nbytes, C.byref(p)) == cb.OK
        assert self.ctx.lib.b2_memset(self.ctx.handle, p, 0, nbytes, self.ctx.stream) == cb.OK
        self.ptrs.append(p.value)
        return p.value

    def array(self, t, n=N):
        a = cb.B2Array()
        a.data = self.zeros(16 * (n + 1))
        a.data2 = self.zeros(64)
        a.length, a.type = n, t
        a.byte_width = FSB_WIDTH if t == cb.FIXED_SIZE_BINARY else 0
        return a

    def out(self):
        a = cb.B2Array()
        self.ptrs.append(a)
        return a

    def free(self):
        lib, h = self.ctx.lib, self.ctx.handle
        lib.b2_sync(h, self.ctx.stream)
        for p in self.ptrs:
            for q in ([p.validity, p.data, p.data2] if isinstance(p, cb.B2Array) else [p]):
                if q:
                    lib.b2_free(h, C.c_void_p(q))


@pytest.fixture
def bufs(ctx):
    b = Bufs(ctx)
    yield b
    b.free()


def expect(st, want):
    """want: None for OK, else (code, message)."""
    got = (st, cb.last_error()) if st != cb.OK else None
    assert got == want


def val(a):
    return cb.B2Value(C.pointer(a), None)


@pytest.mark.parametrize("t", ALL_IDS)
def test_cast(ctx, bufs, t):
    for u in ALL_IDS:
        opt = cb.B2CastOptions(u, 0, 0, 0)
        st = ctx.lib.b2_cast_numeric(ctx.handle, C.byref(bufs.array(t)), C.byref(opt), C.byref(bufs.out()), ctx.stream)
        ok = t in NUMERIC and u in NUMERIC
        expect(st, None if ok else (cb.NOT_IMPLEMENTED, "Unsupported cast from %s to %s using function cast_%s"
                                    % (NAMES.get(t, "?"), NAMES.get(u, "?"), NAMES.get(u, "?"))))


@pytest.mark.parametrize("t", ALL_IDS)
def test_arith_compare_if_else(ctx, bufs, t):
    st = ctx.lib.b2_binary_arith(ctx.handle, cb.ARITH_OPS["add"], val(bufs.array(t)), val(bufs.array(t)), C.byref(bufs.out()),
                                 ctx.stream)
    expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "arithmetic on type id %d" % t))
    st = ctx.lib.b2_compare(ctx.handle, cb.COMPARE_OPS["equal"], val(bufs.array(t)), val(bufs.array(t)), C.byref(bufs.out()),
                            ctx.stream)
    expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "compare on type id %d" % t))
    st = ctx.lib.b2_if_else(ctx.handle, val(bufs.array(cb.BOOL)), val(bufs.array(t)), val(bufs.array(t)), C.byref(bufs.out()),
                            ctx.stream)
    expect(st, None if t in WIDTH or t == cb.BOOL else (cb.NOT_IMPLEMENTED, "if_else over type id %d" % t))


@pytest.mark.parametrize("t", ALL_IDS)
def test_reduce_and_hash_aggregates(ctx, bufs, t):
    r = cb.B2ReduceResult()
    st = ctx.lib.b2_reduce(ctx.handle, C.byref(bufs.array(t)), C.byref(r), ctx.stream)
    expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "sum/mean/min_max over type id %d" % t))
    if st == cb.OK:
        assert r.acc_type == sum_type(t)
    ids = bufs.array(cb.UINT32)
    for kind in ("hash_sum", "hash_product", "hash_variance"):
        agg = C.c_void_p()
        st = ctx.lib.b2_hashagg_create(ctx.handle, cb.HASH_AGG_KINDS[kind], t, None, C.byref(agg))
        expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "hash aggregate over value type id %d" % t))
        if st != cb.OK:
            continue
        try:
            assert ctx.lib.b2_hashagg_out_type(agg) == (cb.DOUBLE if kind == "hash_variance" else sum_type(t))
            assert ctx.lib.b2_hashagg_resize(agg, 1, ctx.stream) == cb.OK
            expect(ctx.lib.b2_hashagg_consume(agg, C.byref(bufs.array(t)), C.byref(ids), ctx.stream), None)
        finally:
            ctx.lib.b2_hashagg_destroy(agg)


@pytest.mark.parametrize("n", [N, 1 << 21])  # 2^21 rows: the partitioned consume
@pytest.mark.parametrize("t", ALL_IDS)
def test_groupby_sumcount(ctx, bufs, t, n):
    for key, value in ((t, cb.INT64), (cb.INT64, t)):
        g = C.c_void_p()
        st = ctx.lib.b2_groupby_sumcount_create(ctx.handle, key, value, 0, C.byref(g))
        if key == t and t not in WIDTH:
            expect(st, (cb.NOT_IMPLEMENTED, "group-by key type id %d" % t))
            continue
        if value == t and t not in NUMERIC:
            expect(st, (cb.NOT_IMPLEMENTED, "group-by value type id %d" % t))
            continue
        expect(st, None)
        try:
            expect(ctx.lib.b2_groupby_sumcount_consume(g, C.byref(bufs.array(key, n)), C.byref(bufs.array(value, n)), ctx.stream), None)
            expect(ctx.lib.b2_groupby_sumcount_merge(g, C.byref(bufs.array(key)), C.byref(bufs.array(sum_type(value))),
                                                     C.byref(bufs.array(cb.INT64)), ctx.stream), None)
            k, s, c = bufs.out(), bufs.out(), bufs.out()
            expect(ctx.lib.b2_groupby_sumcount_finalize(g, C.byref(k), C.byref(s), C.byref(c), ctx.stream), None)
            assert (k.type, s.type, k.length) == (key, sum_type(value), 1)
        finally:
            ctx.lib.b2_groupby_sumcount_destroy(g)


@pytest.mark.parametrize("t", ALL_IDS)
def test_partition_and_sort(ctx, bufs, t):
    counts = (C.c_int64 * 8)()
    st = ctx.lib.b2_range_split(ctx.handle, C.byref(bufs.array(t)), C.byref(bufs.array(t, 1)), 0, 0, C.byref(bufs.out()),
                                C.byref(bufs.out()), counts, ctx.stream)
    expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "b2_range_split: type id %d" % t))
    st = ctx.lib.b2_range_partition(ctx.handle, C.byref(bufs.array(t)), C.byref(bufs.array(t, 1)), 0, C.byref(bufs.out()),
                                    ctx.stream)
    expect(st, None if t in NUMERIC else (cb.NOT_IMPLEMENTED, "b2_range_partition: type id %d" % t))
    st = ctx.lib.b2_sort_indices(ctx.handle, C.byref(bufs.array(t)), 0, 1, C.byref(bufs.out()), ctx.stream)
    expect(st, None if t in NUMERIC or t in BINARY_LIKE else (cb.NOT_IMPLEMENTED, "sort_indices: unsupported type id %d" % t))


@pytest.mark.parametrize("t", ALL_IDS)
def test_take_and_filter(ctx, bufs, t):
    width = FSB_WIDTH if t == cb.FIXED_SIZE_BINARY else WIDTH.get(t, 0)
    fixed_ok = t in BINARY_LIKE or t == cb.BOOL or width in (1, 2, 4, 8, 16)
    st = ctx.lib.b2_take(ctx.handle, C.byref(bufs.array(t)), C.byref(bufs.array(cb.INT64)), 1, C.byref(bufs.out()), ctx.stream)
    expect(st, None if fixed_ok else (cb.NOT_IMPLEMENTED, "take: unsupported value type id %d (width %d)" % (t, width)))
    st = ctx.lib.b2_filter(ctx.handle, C.byref(bufs.array(t)), C.byref(bufs.array(cb.BOOL)), 0, C.byref(bufs.out()), ctx.stream)
    expect(st, None if fixed_ok else (cb.NOT_IMPLEMENTED, "filter: unsupported value type id %d (width %d)" % (t, width)))
    # indices of type t: the fixed-width, boolean and binary Take
    for v in (cb.INT8, cb.INT32, cb.DOUBLE, cb.FIXED_SIZE_BINARY, cb.BOOL, cb.STRING, cb.LARGE_BINARY):
        st = ctx.lib.b2_take(ctx.handle, C.byref(bufs.array(v)), C.byref(bufs.array(t)), 1, C.byref(bufs.out()), ctx.stream)
        expect(st, None if t in INTEGER else (cb.TYPE_ERROR, "take: indices must be an integer array (type id %d)" % t))


@pytest.mark.parametrize("t", ALL_IDS)
def test_take_cast_arith(ctx, bufs, t):
    for to in (cb.FLOAT, cb.DOUBLE):
        other = cb.B2Scalar(0, to, 1)
        oval = cb.B2Value(None, C.pointer(other))
        st = ctx.lib.b2_take_cast_arith(ctx.handle, C.byref(bufs.array(t)), C.byref(bufs.array(cb.INT64)), to,
                                        cb.ARITH_OPS["add"], oval, C.byref(bufs.out()), ctx.stream)
        expect(st, None if t in (cb.DOUBLE, cb.FLOAT, cb.INT64, cb.INT32) else (
            cb.NOT_IMPLEMENTED, "b2_take_cast_arith: float64 / float32 / int64 / int32 values only (type id %d)" % t))
        st = ctx.lib.b2_take_cast_arith(ctx.handle, C.byref(bufs.array(cb.DOUBLE)), C.byref(bufs.array(t)), to,
                                        cb.ARITH_OPS["add"], oval, C.byref(bufs.out()), ctx.stream)
        expect(st, None if t in (cb.INT32, cb.UINT32, cb.INT64, cb.UINT64) else (
            cb.NOT_IMPLEMENTED, "b2_take_cast_arith: 32- or 64-bit indices only (type id %d)" % t))
