"""Host checks of the colliding-key helpers (tests/hash_keys.py) and of the regime model and case table
(tests/grouper_regimes.py) that test_gpu_grouper_edges.py runs: no GPU needed."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import arrow_oracle as ora
from tests import grouper_regimes as gr
from tests import hash_keys as hk
from tests.host_ops import hash64

EDGE_WORDS = [0, 1, 2, 3, (1 << 32) - 1, 1 << 32, (1 << 33) - 1, 1 << 33, (1 << 63) - 1, 1 << 63, (1 << 64) - 2,
              (1 << 64) - 1, 0x5555555555555555, 0xAAAAAAAAAAAAAAAA]


def test_fmix64_round_trip_and_numpy_agreement():
    rng = np.random.default_rng(1)
    words = EDGE_WORDS + [int(x) for x in rng.integers(0, 1 << 63, 2000, dtype=np.int64)] + \
        [int(x) | (1 << 63) for x in rng.integers(0, 1 << 63, 2000, dtype=np.int64)]
    for x in words:
        assert hk.fmix64_inverse(hk.fmix64(x)) == x
        assert hk.fmix64(hk.fmix64_inverse(x)) == x
    arr = np.array(words, np.uint64)
    assert np.array_equal(hk.fmix64_np(arr), hash64(arr))
    assert [int(v) for v in hash64(arr)] == [hk.fmix64(x) for x in words]
    assert np.array_equal(hk.fmix64_inverse_np(hk.fmix64_np(arr)), arr)


def test_constants_read_from_the_sources():
    assert hk.EMPTY_KEY == (1 << 64) - 1 and hk.MAX_PROBE >= 16
    assert hk.PRE_SLOTS & (hk.PRE_SLOTS - 1) == 0 and hk.PART_RADIX & (hk.PART_RADIX - 1) == 0
    assert hk.PRE_PROBE < hk.PRE_SLOTS and hk.DIRECT_MAX_RANGE & (hk.DIRECT_MAX_RANGE - 1) == 0
    assert hk.GUESS_SMALL <= hk.GUESS_FLOOR and hk.GUESS_MID < hk.GUESS_TOP
    assert hk.PART_MIN_ROWS > 0 and hk.SCAN_TILE > 0 and hk.FUSED_PART_CAP >= hk.FUSED_FIRST_CAP


@pytest.mark.parametrize("dtype", [np.int64, np.uint64, np.float64])
def test_built_keys_share_the_requested_bits(dtype):
    fields = hk.slot_field(20) + [(40, 8, 0x3C)]
    keys = hk.keys_with_fields(500, fields, 11, dtype)
    assert keys.dtype == dtype and len(np.unique(keys.view(np.uint64))) == 500
    h = hash64(keys.view(np.uint64))
    assert np.all(h & np.uint64((1 << 20) - 1) == np.uint64(0x5A5A5A5A5A5A5A5A & ((1 << 20) - 1)))
    assert np.all((h >> np.uint64(40)) & np.uint64(0xFF) == np.uint64(0x3C))
    assert not np.any(keys.view(np.uint64) == np.uint64(hk.EMPTY_KEY))
    pre = hk.keys_with_fields(100, hk.pre_slot_field(), 12)
    assert len(set(((hash64(pre.view(np.uint64)) >> np.uint64(20)) & np.uint64(hk.PRE_SLOTS - 1)).tolist())) == 1
    fill = hk.filler_keys(3000, [fields], 13, dtype, exclude=keys)
    hf = hash64(fill.view(np.uint64))
    assert not np.any((hf & np.uint64((1 << 20) - 1) == np.uint64(0x5A5A5A5A5A5A5A5A & ((1 << 20) - 1))) &
                      ((hf >> np.uint64(40)) & np.uint64(0xFF) == np.uint64(0x3C)))
    assert len(np.unique(fill.view(np.uint64))) == 3000
    assert not set(fill.view(np.uint64).tolist()) & set(keys.view(np.uint64).tolist())


def test_consecutive_cluster_fits_a_direct_window():
    keys = hk.consecutive_keys_with_low_bits(300, 14)
    assert np.all(np.diff(keys) > 0) and keys[-1] - keys[0] < hk.DIRECT_MAX_RANGE
    assert len(set((hash64(keys.view(np.uint64)) & np.uint64((1 << 14) - 1)).tolist())) == 1


def test_host_grouper_matches_the_oracle_grouper():
    """the numpy reference the GPU tests use for long batches == oracle.Grouper (first-occurrence ids, uniques, Lookup)"""
    rng = np.random.default_rng(3)
    for t in (pa.int8(), pa.int32(), pa.uint64(), pa.float64()):
        g, og = gr.HostGrouper(t), ora.Grouper([t])
        for b in range(3):
            raw = rng.integers(0, 40, 500).astype(ora.np_dtype(t))
            if b == 2 and t == pa.float64():
                raw[:3] = [np.nan, -0.0, 0.0]
            arr = pa.array(raw, t, mask=rng.random(500) < 0.1)
            assert pa.array(g.consume(arr), pa.uint32()).equals(og.consume(arr))
            assert gr.same_bits(g.get_uniques(), og.get_uniques()[0])
        look = pa.array(rng.integers(0, 60, 300).astype(ora.np_dtype(t)), t, mask=rng.random(300) < 0.1)
        assert g.lookup(look).equals(og.lookup(look))


def test_fused_key_sets_stay_on_target():
    """the fused group-by cases aim at the constants the sources have now: more than kMaxProbe keys on one home slot of
    the tables they start from, equal radix digits, more than kPreProbe keys on one pre-aggregation slot"""
    c, _, fill = gr.fused_atomic_keys()
    assert len(c) > hk.MAX_PROBE and gr.fused_atomic_grows(c) >= 3
    h = hash64(c.view(np.uint64))
    assert len(set((h & np.uint64(hk.FUSED_FIRST_CAP - 1)).tolist())) == 1
    c, pre, fill = gr.fused_partitioned_keys()
    h, hp = hash64(c.view(np.uint64)), hash64(pre.view(np.uint64))
    assert len(c) > hk.MAX_PROBE
    for cap in (hk.FUSED_PART_CAP, 2 * hk.FUSED_PART_CAP):   # parked at the first table, replayed into the next one
        assert len(set((h & np.uint64(cap - 1)).tolist())) == 1
    digits = np.uint64(hk.PART_RADIX * hk.PART_RADIX - 1)   # the digits of both radix passes
    assert len(set((h & digits).tolist())) == 1 and len(set((hp & digits).tolist())) == 1
    assert len(pre) > hk.PRE_PROBE
    assert len(set(((hp >> np.uint64(20)) & np.uint64(hk.PRE_SLOTS - 1)).tolist())) == 1
    hf = hash64(fill.view(np.uint64))
    assert not np.any((hf & np.uint64(2 * hk.FUSED_PART_CAP - 1)) == h[0])


def test_case_tables_reach_every_regime():
    """the GPU case tables still reach every branch of grouper_run they were built for (fails after a retune that moves
    a case off its target)"""
    narrow = gr.narrow_cases()
    direct = {k: (t, True, b) for k, (t, b) in gr.direct_cases().items()}
    models = gr.run_model({**narrow, **direct})
    for case, batch, key, value in gr.expected_outcomes():
        got = models[case].log[batch][key]
        assert got == value, f"{case} batch {batch}: {key} = {got}, want {value}"
    modes = {o["mode"] for m in models.values() for o in m.log}
    flags = {o["flag"] for m in models.values() for o in m.log}
    assert modes == {"direct", "hash"} and {"slots", "rows"} <= flags
    # every clustered case makes its device table overflow at least once, and the fallback case's stored uniques
    # overflow grouper_rebuild itself
    assert sum(o["regrows"] for m in models.values() for o in m.log) >= 10
    assert any(o["rehash_overflows"] for m in models.values() for o in m.log)
