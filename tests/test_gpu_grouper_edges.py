"""The Grouper (grouper.cu, grouper_wide.cu), its consumers (hash join, unique / value_counts / dictionary_encode,
count_distinct) and the fused group-by (groupby_fused.cu) on keys BUILT to collide (tests/hash_keys.py): probe limits,
table regrowth, rehash overflow, the two special slots (the all-ones key and null), the direct-addressed window's edges,
the narrow / wide key encodings.  Every result is compared exactly -- ids, not ids up to a bijection -- with
tests/grouper_regimes.HostGrouper, oracle.Grouper, oracle.hash_join_indices or the oracle's vector-hash functions;
test_hash_keys_regimes.py checks on the host that the cases still reach the regimes they were built for."""
import functools

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from oracle import arrow_oracle as ora
from tests import grouper_regimes as gr
from tests import hash_keys as hk
from tests.util import assert_equal

pytestmark = pytest.mark.gpu
JOIN_TYPES = ["inner", "left outer", "left semi", "left anti", "full outer"]


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


@functools.lru_cache(maxsize=None)
def narrow():
    return gr.narrow_cases()


@functools.lru_cache(maxsize=None)
def direct():
    return gr.direct_cases()


def run_grouper(ctx, t, batches, lookups=()):
    """consume every batch on the device and on the host reference; ids, uniques and num_groups must agree after each.
    Returns the grouper, the reference and the device's outputs (ids and uniques per batch, then the Lookup results)."""
    g, ref = bc.Grouper([t], ctx), gr.HostGrouper(t)
    outs = []
    for b, keys in enumerate(batches):
        ids = g.consume(dev(keys, ctx)).to_arrow()
        want = pa.array(ref.consume(keys), pa.uint32())
        assert_equal(ids, want, f"{t} batch {b}")
        assert g.num_groups == len(ref.uniques)
        uniq = g.get_uniques()[0].to_arrow()
        assert gr.same_bits(uniq, ref.get_uniques()), f"uniques after batch {b}"
        outs += [ids, uniq]
    for look in lookups:
        got = g.lookup(dev(look, ctx)).to_arrow()
        assert_equal(got, ref.lookup(look), "lookup")
        outs.append(got)
    return g, ref, outs


def neighbours(t, n=200):
    """keys in the clustered neighbourhoods (the same low 16 / 24 bits) that the cases never insert, the special keys, null"""
    words = np.concatenate([gr.cluster(n, 16, 101).view(np.uint64), gr.cluster(n, 24, 102).view(np.uint64),
                            np.array([hk.EMPTY_KEY, 0], np.uint64)])
    mask = np.zeros(len(words) + 1, bool)
    mask[-1] = True
    return pa.array(np.concatenate([words, np.zeros(1, np.uint64)]).view(ora.np_dtype(t)), t, mask=mask)


@pytest.mark.parametrize("name", [
    "first_small", "first_large", "later_batch", "special_in_cluster", "flag_slots_special", "flag_rows_special",
    "flag_rows_special_ends",
    "load_rebuild", "fallback_rehash"])
def test_narrow_hash_table_regimes(ctx, name, monkeypatch):
    t, direct_on, batches = narrow()[name]
    if not direct_on:
        monkeypatch.setenv("B2_GROUPER_DIRECT", "0")
    stored = pa.concat_arrays([b.slice(0, 300) for b in batches])
    run_grouper(ctx, t, batches, [neighbours(t), stored])


def test_lookup_before_consume_and_after_reset(ctx, monkeypatch):
    for direct_on in (True, False):
        monkeypatch.setenv("B2_GROUPER_DIRECT", "1" if direct_on else "0")
        for t in (pa.int64(), pa.uint64()):
            look = neighbours(t)
            g = bc.Grouper([t], ctx)
            got = g.lookup(dev(look, ctx)).to_arrow()
            assert got.null_count == len(look)
            batch = narrow()["flag_rows_special"][2][3] if t == pa.uint64() else narrow()["first_small"][2][0]
            ref = gr.HostGrouper(t, direct_on)
            assert_equal(g.consume(dev(batch, ctx)).to_arrow(), pa.array(ref.consume(batch), pa.uint32()))
            assert_equal(g.lookup(dev(look, ctx)).to_arrow(), ref.lookup(look))
            g.reset()
            assert g.num_groups == 0
            assert g.lookup(dev(look, ctx)).to_arrow().null_count == len(look)
            # after a reset the ids start again from 0, in this batch's first-occurrence order
            ref = gr.HostGrouper(t, direct_on)
            assert_equal(g.consume(dev(look, ctx)).to_arrow(), pa.array(ref.consume(look), pa.uint32()))
            assert gr.same_bits(g.get_uniques()[0].to_arrow(), ref.get_uniques())


def _ord_to_value(t, o):
    """the key whose order-preserving encoding (bits ^ sign flip) is o"""
    w = np.dtype(ora.np_dtype(t)).itemsize
    return int(np.array([(o ^ gr.SIGN_FLIP.get(t, 0)) & ((1 << 8 * w) - 1)], {1: np.uint8, 2: np.uint16, 4: np.uint32,
                                                                            8: np.uint64}[w]).view(ora.np_dtype(t))[0])


@pytest.mark.parametrize("name", ["roomy_n4000_below", "roomy_n4000_at", "roomy_n10000_below", "roomy_n10000_at",
                                  "widen_to_limit", "reseat_below_above", "int8_full", "int16_ends", "int32_ends",
                                  "int64_ends", "int64_min", "uint64_top", "all_null_first"])
def test_direct_window_edges(ctx, name, monkeypatch):
    t, batches = direct()[name]
    model = gr.HostGrouper(t)
    for b in batches:
        model.consume(b)
    # the keys just outside and just inside the last direct window, when it is still direct
    looks = [pa.concat_arrays(batches).slice(0, 500), pa.array([None], t)]
    edge = []
    for o in model.log:
        if o["mode"] == "direct":
            for ordv in (o["lo"] - 1, o["lo"], o["lo"] + o["dcap"] - 1, o["lo"] + o["dcap"]):
                if 0 <= ordv <= hk.M64 and (np.dtype(ora.np_dtype(t)).itemsize == 8 or ordv < 1 << (8 * np.dtype(ora.np_dtype(t)).itemsize)):
                    edge.append(_ord_to_value(t, ordv))
    if edge:
        looks.append(pa.array(np.array(edge, ora.np_dtype(t)), t))
    direct_out = run_grouper(ctx, t, batches, looks)[2]
    monkeypatch.setenv("B2_GROUPER_DIRECT", "0")
    hash_out = run_grouper(ctx, t, batches, looks)[2]
    # the device in direct mode and in hash mode: the same ids, uniques and Lookup results
    assert len(direct_out) == len(hash_out)
    for a, b in zip(direct_out, hash_out):
        assert gr.same_bits(a, b)


def check_oracle_grouper(ctx, types, batches, lookups):
    g, og = bc.Grouper(types, ctx), ora.Grouper(types)
    for b, cols in enumerate(batches):
        assert_equal(g.consume([dev(c, ctx) for c in cols]).to_arrow(), og.consume(cols), f"batch {b}")
        for got, want in zip(g.get_uniques(), og.get_uniques()):
            assert_equal(got.to_arrow(), want, f"uniques after batch {b}")
    for cols in lookups:
        assert_equal(g.lookup([dev(c, ctx) for c in cols]).to_arrow(), og.lookup(cols), "lookup")


def _col(t, n, seed, lo, hi, offset, nulls=0.2):
    rng = np.random.default_rng(seed)
    v = rng.integers(lo, hi, n + offset, endpoint=True).astype(ora.np_dtype(t))
    return pa.array(v, t, mask=rng.random(n + offset) < nulls).slice(offset)


@pytest.mark.parametrize("types", [
    [pa.int32(), pa.int16(), pa.int8()],                 # 56 value bits + 3 null bits: narrow
    [pa.uint8()] * 7,                                    # 56 + 7 = 63 bits: narrow
    [pa.int32(), pa.int32()],                            # 64 + 2: wide
    [pa.uint8()] * 8,                                    # 64 + 8: wide
], ids=lambda ts: "+".join(str(t) for t in ts))
def test_multi_column_encoding_boundary(ctx, types):
    n = 3000

    def batch(seed):   # every column sliced at its own non-multiple-of-8 offset; values at the type's ends and 0
        cols = []
        for j, t in enumerate(types):
            info = np.iinfo(ora.np_dtype(t))
            off = 3 + 5 * j
            c = _col(t, n + off, seed + j, 0, 2, 0)
            ends = np.array([info.min, 0, info.max], ora.np_dtype(t))
            cols.append(pa.array(ends[ora.values(c)], t, mask=~ora.validity(c)).slice(off))
            assert cols[-1].offset == off
        return cols

    # tuples that differ only in which column is null, and null vs 0 in the same column
    k = len(types)
    crafted = []
    for j, t in enumerate(types):
        vals = np.zeros(2 * k, ora.np_dtype(t))
        mask = np.zeros(2 * k, bool)
        mask[j] = True          # row j: column j null, every other column 0
        crafted.append(pa.array(vals, t, mask=mask))
    check_oracle_grouper(ctx, types, [crafted, batch(1), batch(2)], [batch(3), crafted])


def words_at(t, lens, seed, nulls=None, alphabet=b"ab"):
    rng = np.random.default_rng(seed)
    vals = [bytes(rng.choice(list(alphabet), int(L)).tolist()) for L in lens]
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        vals = [v.decode() for v in vals]
    return pa.array([None if nulls is not None and nulls[i] else v for i, v in enumerate(vals)], t)


@pytest.mark.parametrize("st", [pa.string(), pa.large_string(), pa.large_binary()], ids=str)
def test_wide_keys_record_tail_edges_and_partial_unknowns(ctx, st):
    rng = np.random.default_rng(7)
    n = 2000
    lens = rng.choice([0, 1, 26, 27, 28, 29, 30, 60], n)
    s1 = words_at(st, lens, 1, rng.random(n) < 0.05)
    s2 = words_at(st, rng.choice([27, 28, 29], n), 2, rng.random(n) < 0.05)
    i1 = pa.array(rng.integers(0, 4, n) * (1 << 40), pa.int64(), mask=rng.random(n) < 0.05)
    # "", "\0" and null: three different keys; strings equal in the 28-byte record head, different in the tail
    zero = "\0" if pa.types.is_string(st) or pa.types.is_large_string(st) else b"\0"
    empty = "" if pa.types.is_string(st) or pa.types.is_large_string(st) else b""
    head = "h" * 28 if pa.types.is_string(st) or pa.types.is_large_string(st) else b"h" * 28
    tails = [head + ("x" if isinstance(head, str) else b"x"), head + ("y" if isinstance(head, str) else b"y"), head]
    specials = pa.array([empty, zero, None] + tails, st)
    m = len(specials)
    b1 = [pa.concat_arrays([specials, s1]).slice(0), pa.concat_arrays([pa.array([3] * m, pa.int64()), i1]),
          pa.concat_arrays([pa.array([empty] * m, st), s2])]
    b1 = [c.slice(k) for k, c in enumerate(b1)]   # each column at its own offset
    b1 = [c.slice(0, len(b1[-1])) for c in b1]
    b2 = [c.slice(500, 800) for c in b1]
    # lookup rows where exactly one of the three parts is unknown
    unk = words_at(st, [28] * 600, 99, alphabet=b"xyz")
    l0, l1, l2 = (c.slice(0, 600) for c in b1)
    look = [[unk, l1, l2], [l0, pa.array(np.full(600, 5, np.int64)), l2], [l0, l1, unk], [l0, l1, l2]]
    check_oracle_grouper(ctx, [st, pa.int64(), st], [b1, b2], look)


def test_wide_lookup_under_one_bit_hashes(ctx, monkeypatch):
    """with 1-bit hashes about half of all unknown strings share their hash with the one stored string: the byte
    comparison must make them null.  One stored string cannot collide with another, so the Consume keeps the 1-bit hash
    (two colliding stored strings would make it reseed with a wider hash)."""
    monkeypatch.setenv("B2_GROUPER_HASH_BITS", "1")
    for st in (pa.string(), pa.large_binary()):
        enc = (lambda s: s) if pa.types.is_string(st) else (lambda s: s.encode())
        head = "h" * 28   # equal 28-byte record heads: only the tail in the byte store tells these apart
        stored = pa.array([enc(head + "aa")], st)
        # same length and head, other tail; and strings of other lengths that differ only in the head or the tail
        letters = "bcdefghijklmnopqrstuvwxyz"
        unknown = pa.array([enc(head + a + b) for a in "ab" for b in letters] +
                           [enc(head + a) for a in letters] + [enc("g" + head[1:] + "aa"), enc(head + "aaa")], st)
        assert len(unknown) >= 64
        check_oracle_grouper(ctx, [st], [[stored]], [[unknown], [pa.concat_arrays([unknown, stored])]])
        # the same-head strings consumed as new keys: each gets its own group whatever the hashes did
        check_oracle_grouper(ctx, [st], [[stored], [pa.concat_arrays([stored, unknown])]], [[unknown]])


# ---- consumers ----------------------------------------------------------------------------------------------------
def check_join(ctx, left, right, join_type):
    got_l, got_r = bc.hash_join_indices([dev(k, ctx) for k in left], [dev(k, ctx) for k in right], join_type)
    want_l, want_r = ora.hash_join_indices(left, right, join_type)
    assert_equal(got_l.to_arrow(), want_l, join_type)
    if want_r is None:
        assert got_r is None
    else:
        assert_equal(got_r.to_arrow(), want_r, join_type)


@functools.lru_cache(maxsize=None)
def join_sides():
    """right: 300 clustered keys (the first 100 on one row each, the rest on 2..4 rows) + fillers, so its grouper
    overflows and regrows; left: the right keys, their never-inserted neighbours and nulls"""
    rng = np.random.default_rng(21)
    c = gr.cluster(300, 16, 1)
    fill = hk.filler_keys(500, [hk.slot_field(16)], 22, exclude=c)
    right = np.concatenate([c[:100], np.repeat(c[100:], rng.integers(2, 5, 200)), fill])
    rng.shuffle(right)
    pool = np.concatenate([c, fill, gr.cluster(300, 16, 101)])
    return right, pool


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_join_clustered_right_side_and_scan_tile_lengths(ctx, join_type):
    right, pool = join_sides()
    rng = np.random.default_rng(23)
    r = pa.array(right, pa.int64(), mask=rng.random(len(right)) < 0.02)
    for n in (hk.SCAN_TILE - 1, hk.SCAN_TILE, hk.SCAN_TILE + 1, 65535, 65536, 65537):
        left = pa.array(rng.choice(pool, n), pa.int64(), mask=rng.random(n) < 0.03)
        check_join(ctx, [left], [r], join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_join_direct_window_multi_column_and_all_null(ctx, join_type):
    rng = np.random.default_rng(24)
    # direct-mode right side: keys [1000, 1999]; left keys one outside its window (lo - 1, lo + cap) on both sides, at
    # the window's ends, in its empty padding (999, 2000) and on stored keys
    r = pa.array(np.concatenate([np.arange(1000, 2000), np.arange(1000, 1100)]).astype(np.int32))
    model = gr.HostGrouper(pa.int32())
    model.consume(r)
    w = model.log[0]
    assert w["mode"] == "direct" and w["lo"] < 999 + (1 << 31) and w["lo"] + w["dcap"] > 2000 + (1 << 31)
    edges = [_ord_to_value(pa.int32(), o) for o in (w["lo"] - 1, w["lo"], w["lo"] + w["dcap"] - 1, w["lo"] + w["dcap"])]
    left = pa.array(rng.choice(np.array(edges + [999, 1000, 1500, 1999, 2000], np.int32), 5000))
    check_join(ctx, [left], [r], join_type)
    # a null in just one column of a two-column key, on either side; each column sliced at its own offset
    def side(n, seed):
        a = _col(pa.int16(), n, seed, 0, 5, 3, 0.1)
        b = _col(pa.int64(), n, seed + 1, 0, 5, 7, 0.1)
        return [a, b]
    check_join(ctx, side(3000, 25), side(2000, 27), join_type)
    # an all-null right side
    check_join(ctx, [left], [pa.array([None] * 300, pa.int32())], join_type)


@pytest.mark.parametrize("name", ["first_small", "special_in_cluster", "flag_rows_special"])
def test_vector_hash_over_clustered_and_special_keys(ctx, name):
    batches = narrow()[name][2]
    v = pa.concat_arrays(batches)
    dv = dev(v, ctx)
    assert gr.same_bits(bc.unique(dv).to_arrow(), ora.unique(v))
    vals, counts = bc.value_counts(dv)
    want = ora.value_counts(v)
    assert gr.same_bits(vals.to_arrow(), want.field("values"))
    assert counts.to_arrow().equals(want.field("counts"))
    for enc in ("mask", "encode"):
        got = bc.dictionary_encode(dv, enc).to_arrow()
        w = ora.dictionary_encode(v, enc)
        assert got.indices.equals(w.indices), enc
        assert gr.same_bits(got.dictionary, w.dictionary), enc
    u = ora.unique(v)
    for mode, want_n in (("only_valid", len(u) - u.null_count), ("only_null", u.null_count), ("all", len(u))):
        assert bc.count_distinct(dv, mode).as_py() == want_n


# ---- the fused group-by ----------------------------------------------------------------------------------------------
def fused_reference(keys: pa.Array, values: pa.Array):
    """{key bits or None: (sum mod 2^64 or None, count)} over the valid values"""
    kb, kv = gr.key_bits(keys)
    vb, vv = ora.values(values).view(np.uint64), ora.validity(values)
    u, inv = np.unique(kb[kv], return_inverse=True)
    gid = np.full(len(kb), len(u), np.int64)   # the null key is group len(u)
    gid[kv] = inv.reshape(-1)
    sums = np.zeros(len(u) + 1, np.uint64)
    with np.errstate(over="ignore"):
        np.add.at(sums, gid[vv], vb[vv])
    cnt = np.bincount(gid[vv], minlength=len(u) + 1)
    names = [int(x) for x in u] + [None]
    present = np.bincount(gid, minlength=len(u) + 1) > 0
    return {names[j]: (int(sums[j]) if cnt[j] else None, int(cnt[j])) for j in range(len(u) + 1) if present[j]}


def check_fused(ctx, keys, values, want_paths):
    gb = bc.GroupBySumCount(pa.int64(), pa.int64(), ctx=ctx)
    gb.consume(dev(keys, ctx), dev(values, ctx))
    assert {k: v for k, v in gb.path_counts().items() if v} == want_paths
    k, s, c = (x.to_arrow() for x in gb.finalize())
    kb, kv = gr.key_bits(k)
    sb, sv = ora.values(s).view(np.uint64), ora.validity(s)
    got = {(int(kb[i]) if kv[i] else None): (int(sb[i]) if sv[i] else None, int(ora.values(c)[i])) for i in range(len(k))}
    assert len(got) == len(k), "a key was emitted twice"
    assert got == fused_reference(keys, values)


def fused_rows(n, seed, clustered, pre, fill):
    rng = np.random.default_rng(seed)
    pick = rng.random(n)
    keys = np.where(pick < 0.7, rng.choice(clustered, n), np.where(pick < 0.8, rng.choice(pre, n), rng.choice(fill, n)))
    keys[rng.choice(n, 50, replace=False)] = -1          # the all-ones key
    keys[0], keys[-1] = -1, clustered[0]
    kmask = rng.random(n) < 0.001
    kmask[1] = True
    vals = pa.array(rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64), mask=rng.random(n) < 0.05)
    return pa.array(keys, pa.int64(), mask=kmask), vals


def test_fused_atomic_path_grow_and_retry_pending(ctx):
    """below kPartMinRows rows: kMaxProbe + 44 keys on one home slot in every table up to 16x the first size; the table
    grows until they fit, each round retrying only the rows that did not (gr.fused_atomic_keys)"""
    c, pre, fill = gr.fused_atomic_keys()
    keys, vals = fused_rows(hk.PART_MIN_ROWS // 10, 33, c, pre, fill)
    check_fused(ctx, keys, vals, {"atomic": 1})


def test_fused_partitioned_path_parks_and_replays(ctx):
    """at kPartMinRows rows: kMaxProbe + 44 keys share one home slot in the first two partitioned-path tables and both
    radix digits; 2 * kPreProbe + 4 keys share both digits and one pre-aggregation slot, so their rows spill past shared
    memory; the entries that meet the full neighbourhood are parked and replayed into larger tables
    (gr.fused_partitioned_keys)"""
    c, pre, fill = gr.fused_partitioned_keys()
    keys, vals = fused_rows(hk.PART_MIN_ROWS + 7, 44, c, pre, fill)
    check_fused(ctx, keys, vals, {"general": 1})
