"""CPU checks of tests/packed_regimes.py: the restatement agrees with the constants it reads, every case of
test_gpu_groupby_packed_edges.py reaches the regime it is named for, and the exact reference agrees with pyarrow."""
import numpy as np
import pyarrow as pa
import pytest

from . import packed_regimes as P


def test_constants_and_fields():
    assert P.K_DENSE_MAX_RANGE == 1 << 24 and P.K_PART_MIN_ROWS == 1 << 21 and P.DENSE_MIN_ROWS == 1 << 22
    assert P.K_SLICE_TUPLES == P.K_CCHUNK * P.K_CSLICE_CHUNKS == 8192
    assert P.DEFAULT_BAND_BYTES // 8 == 3_145_728 and P.SAMPLE_ROWS == 65536
    # m = (63 - vb) / 2: the count field keeps m + 1 bits and the sum field vb + m bits of a 64-bit word
    for vb in range(1, 63):
        m = (P.M_NUM - vb) // 2
        assert 64 - (vb + m) >= m + 1
        assert (1 << m) * ((1 << vb) - 1) < 1 << (vb + m)
    # the dense limit: vb = 19 is the widest window whose sub-batches hold 2^22 rows
    assert (P.M_NUM - 19) // 2 == P.M_MIN and (P.M_NUM - 20) // 2 < P.M_MIN
    for vt, m in ((pa.int8(), 27), (pa.uint8(), 27), (pa.int16(), 23), (pa.uint16(), 23)):
        w = P.value_window(np.zeros(1, P.np_dtype(vt)), None, np.arange(1), 62)
        assert w.vb == vt.bit_width and (P.M_NUM - w.vb) // 2 == m
    assert P.dense_fields(P.Window(32, 0), 1 << 22, 10, P.DEFAULT_BAND_BYTES) is None
    # NARROW: 32-bit partial sums of one slice of top values fit at vb = 19 and not at vb = 20
    assert P.K_SLICE_TUPLES * ((1 << P.NARROW_VB_MAX) - 1) < 1 << 32 <= P.K_SLICE_TUPLES * ((1 << (P.NARROW_VB_MAX + 1)) - 1)
    assert P.NARROW_KB_MAX == 31  # 32-bit keys with the all-ones empty marker


def test_value_window_is_centred_and_capped():
    n = 1 << 20
    v = np.full(n, 1000, np.int64)
    v[0], v[16] = -1000, 1000
    w = P.value_window(v, None, P.sample_rows(n), 62)
    rng = 2000
    assert w.vb == max(8, rng.bit_length() + 2)
    lo, hi = w.lo(pa.int64()), w.hi(pa.int64())
    assert hi - lo == (1 << w.vb) - 1 and lo < -1000 and hi > 1000 and abs((1000 - hi) - (lo + 1000)) <= 1
    assert P.value_window(v, None, P.sample_rows(n), 11).vb == 11   # need = 11: cut to the cap
    assert P.value_window(v, None, P.sample_rows(n), 10) is None    # the cap below the sampled range


@pytest.mark.parametrize("case", P.fused_cases(), ids=lambda c: c.name)
def test_fused_case_reaches_its_regime(case):
    plans, batches = case.plans()
    assert [p.path for p in plans] == case.paths, [p.why for p in plans]
    if case.check:
        case.check(plans, batches)


@pytest.mark.parametrize("case", P.byid_cases(), ids=lambda c: c.name)
def test_hash_sum_case_reaches_its_regime(case):
    plans, _ = case.plans()
    assert [p.dense is not None for p in plans] == case.dense, [p.why for p in plans]


def test_fused_field_cases_fill_their_fields():
    cases = {c.name: c for c in P.fused_cases()}
    # the int16 hot key: 2^23 top values in sub-batch 0 fill the sum field to 2^(vb + m) - 2^m
    c = cases["dense_hot_int16"]
    plans, b = c.plans()
    d = plans[0].dense
    vp = P.value_bits(b[0].vals[:d.sub]) - np.uint64(d.window.vbase)
    assert int(vp.astype(object).sum()) == (1 << d.m) * ((1 << d.window.vb) - 1)
    assert b[0].keys[:2 * d.sub].min() == b[0].keys[:2 * d.sub].max()
    # the compact cases: kb + vb + 1 == 64 where the name says so
    for name in ("compact_kb40_vb23_full", "compact_kb42_vb_cut_to_21", "compact_kb31_int32_values_full"):
        p = cases[name].plans()[0][0].compact
        assert p.kb + p.window.vb + 1 == 64, name
    assert cases["compact_kb31_vb19_narrow"].plans()[0][0].compact.narrow
    for name in ("compact_kb31_vb20_wide", "compact_kb32_vb19_wide", "compact_kb23_vb40_wide_carry"):
        assert not cases[name].plans()[0][0].compact.narrow, name


def _pyarrow_group_by(keys, kvalid, vals, vvalid, kt, vt):
    import pyarrow.acero  # noqa: F401
    t = pa.table({"k": pa.array(keys, kt, mask=None if kvalid is None else ~kvalid),
                  "v": pa.array(vals, vt, mask=None if vvalid is None else ~vvalid)})
    return t.group_by("k", use_threads=False).aggregate([("v", "sum"), ("v", "count")]).sort_by("k")


@pytest.mark.parametrize("kt", P.INT_TYPES, ids=str)
@pytest.mark.parametrize("vt", P.INT_TYPES, ids=str)
def test_reference_matches_pyarrow(kt, vt):
    rng = np.random.default_rng(kt.bit_width * 31 + vt.bit_width + P.signed(kt) * 7 + P.signed(vt))
    n = 4000
    ki, vi = np.iinfo(P.np_dtype(kt)), np.iinfo(P.np_dtype(vt))
    keys = rng.integers(ki.min, ki.max, n, dtype=P.np_dtype(kt), endpoint=True)
    keys[: n // 2] = keys[rng.integers(0, 40, n // 2)]            # repeated keys
    keys[:3] = [ki.min, ki.max, ki.max]
    vals = rng.integers(vi.min, vi.max, n, dtype=P.np_dtype(vt), endpoint=True)
    vals[:200] = vi.max                                           # sums that wrap
    kvalid, vvalid = rng.random(n) >= 0.05, rng.random(n) >= 0.1
    vvalid[keys == keys[5]] = False                               # a group whose values are all null
    got = P.group_sum_count(keys, kvalid, vals, vvalid, kt, vt)
    want = _pyarrow_group_by(keys, kvalid, vals, vvalid, kt, vt)
    assert got["k"].combine_chunks().equals(want["k"].combine_chunks())
    assert got["count"].combine_chunks().equals(want["v_count"].combine_chunks())
    assert got["sum"].combine_chunks().equals(want["v_sum"].combine_chunks().cast(got["sum"].type))


def test_reference_sum_by_id_matches_pyarrow():
    rng = np.random.default_rng(5)
    n, groups = 5000, 300
    ids = rng.integers(0, groups - 3, n, dtype=np.uint32)
    for vt in (pa.int64(), pa.uint64(), pa.int8()):
        info = np.iinfo(P.np_dtype(vt))
        vals = rng.integers(info.min, info.max, n, dtype=P.np_dtype(vt), endpoint=True)
        vvalid = rng.random(n) >= 0.1
        got = P.sum_by_id(ids, vals, vvalid, groups, vt)
        import pyarrow.acero  # noqa: F401
        t = pa.table({"g": pa.array(ids), "v": pa.array(vals, vt, mask=~vvalid)}).group_by("g", use_threads=False) \
            .aggregate([("v", "sum")])
        want = [None] * groups
        for g, s in zip(t["g"].to_pylist(), t["v_sum"].to_pylist()):
            want[g] = s
        assert got.to_pylist() == want
