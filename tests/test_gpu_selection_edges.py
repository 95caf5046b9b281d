"""Filter and Take on the device at the edges of their kernels, compared byte for byte with tests/selection_ref.py (pinned
to pyarrow by test_selection_edges_oracle.py): validity equal, and the bytes of every valid row equal, so a kernel that
canonicalised a NaN payload or turned -0.0 into +0.0 fails.  Every result also has its null_count checked and passes
Arrow's full validation.

The kernel constants are read from the sources, and the inputs are placed where the host and the kernels change regime:
- fixed-width Filter (selection_filter.cu) at byte widths 1, 2, 4, 8 and 16: the 512-row chunk and its dense-chunk
  threshold (kChunkRows / 8 survivors), the sparse / dense template choice (out_len < n / 8), the span of kSpanTiles tiles
  of the chained scan and a look-back longer than one 32-cell step, 16-byte aligned and unaligned values, unaligned masks;
- fixed-width Take (selection_take.cu) at every width x the eight index types: lengths k * (32 * V * kUnroll) +- 1, index
  offsets that force the scalar path, the first bad row of several reported, L2 validity bands, the partitioned path;
- bool Filter / Take (selection_bool.cu) with the output tile starting at every bit of a 64-bit word;
- utf8 / binary Filter / Take (selection_binary.cu): tiles whose output needs a coarse index above 2^6 bytes, empty rows
  at 16-byte output boundaries, kTakeTile +- 1 indices, data buffers off 8-byte alignment, dictionaries;
- the int32-offset capacity: Take refuses more than 2^31 - 2 output bytes, Filter keeps an input of 2^31 - 1.
test_case_tables_reach_every_regime restates the host's choices from each case's inputs and fails if an edit of the
tables drops a regime."""
import gc
import os
import re

import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray
from tests import selection_ref as sr
from tests.test_selection_edges_oracle import (INDEX_TYPES, STRING_TYPES, bitmap, bool_array, dictionary_array,
                                              fixed_array, in_range_bytes, index_array)
from tests.util import SEED, random_array

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constant(text, name):
    return int(re.search(rf"constexpr int {name} = (\d+);", text).group(1))


_COMMON, _FILTER = _source("common.cuh"), _source("selection_filter.cu")
assert "constexpr int kWarpsPerBlock = kBlock / 32;" in _COMMON
TILE = _constant(_source("selection.cuh"), "kTileRows")
CHUNK = _constant(_FILTER, "kChunkRows")
SPAN_TILES = _constant(_FILTER, "kSpanTiles")
UNROLL = _constant(_source("elementwise.cuh"), "kUnroll")
WARPS = _constant(_COMMON, "kBlock") // 32
TAKE_TILE = _constant(_source("selection_binary.cu"), "kTakeTile")
SPAN = SPAN_TILES * TILE
LOOKBACK_STEP = 32  # a look-back step reads one predecessor cell per lane

W_LAYOUTS = {1: [pa.int8(), pa.binary(1)], 2: [pa.float16(), pa.binary(2)],
             4: [pa.int32(), pa.date32(), pa.binary(4)], 8: [pa.float64(), pa.timestamp("us", tz="UTC"), pa.binary(8)],
             16: [pa.binary(16)]}
FILTER_LAYOUTS = [t for ts in W_LAYOUTS.values() for t in ts]
TAKE_LAYOUTS = [pa.int8(), pa.binary(1), pa.float16(), pa.binary(2), pa.date32(), pa.binary(4), pa.float64(),
                pa.timestamp("ns"), pa.binary(8), pa.binary(16)]
FILTER_LENGTHS = [1, CHUNK - 1, CHUNK, CHUNK + 1, TILE - 1, TILE, TILE + 1, SPAN - 1, SPAN + 1,
                  33 * SPAN - 1, 33 * SPAN + 1, 70 * SPAN + 123]
MASK_KINDS = ["all_true", "all_false", "span_last", "chunk_edge", "last_partial_chunk", "below_n8", "at_n8", "random",
              "all_null"]
VALUE_OFFSETS = (0, 1, 16)  # 16 rows keep 16-byte alignment at every width; 1 row breaks it below width 16
MASK_OFFSETS = (0, 3, 13)
VALIDITY = ("none", "present", "unknown")  # no bitmap; a bitmap with its null count; a bitmap with null_count = -1


def gpu(f):
    return pytest.mark.gpu(f)


# ---- case tables ------------------------------------------------------------------------------------------------------
def filter_cases(t):
    """(n, kind, null_selection, mask null share, validity, values offset, mask offset) for layout t; the rotations make
    each length meet each setting"""
    cases, k = [], 0
    for n in FILTER_LENGTHS:
        for kind in MASK_KINDS:
            cases.append((n, kind, (sr.DROP, sr.EMIT_NULL)[k % 2], (0.0, 0.2, 0.05)[k % 3], VALIDITY[(k // 2) % 3],
                          VALUE_OFFSETS[(k // 3) % 3], MASK_OFFSETS[(k // 2) % 3]))
            k += 1
    return cases


def selection(kind, n, rng) -> np.ndarray:
    """the rows a mask kind keeps"""
    sel = np.zeros(n, bool)
    if kind == "all_true":
        sel[:] = True
    elif kind == "span_last":  # the last row of every span (of the array, for the final partial span)
        sel[np.minimum(np.arange(SPAN - 1, n + SPAN - 1, SPAN), n - 1)] = True
    elif kind == "chunk_edge":  # kChunkRows / 8 - 1 and kChunkRows / 8 survivors in alternate chunks
        for c0 in range(0, n, CHUNK):
            m = min(CHUNK, n - c0)
            sel[c0 + rng.choice(m, min(m, CHUNK // 8 - 1 + (c0 // CHUNK) % 2), replace=False)] = True
    elif kind == "last_partial_chunk":
        sel[(n - 1) // CHUNK * CHUNK:] = True
    elif kind in ("below_n8", "at_n8"):
        sel[rng.choice(n, max(n // 8 - (kind == "below_n8"), 0), replace=False)] = True
    elif kind == "random":
        sel = rng.random(n) < 0.5
    return sel


def mask_array(sel, null_selection, null_p, offset, rng, all_null=False) -> pa.Array:
    """a bool mask (sliced at `offset`) that keeps exactly `sel` under null_selection; a share null_p of the rows is null
    (rows the null rule keeps anyway), with random data bits under the nulls"""
    n = len(sel)
    m = n + offset
    data, valid = rng.random(m) < 0.5, np.ones(m, bool)
    null = np.ones(n, bool) if all_null else ((~sel if null_selection == sr.DROP else sel) & (rng.random(n) < null_p))
    valid[offset:] = ~null
    data[offset:] = np.where(null, data[offset:], sel)
    bufs = [bitmap(valid) if (all_null or null_p > 0) else None, bitmap(data)]
    arr = pa.Array.from_buffers(pa.bool_(), m, bufs, null_count=-1 if bufs[0] is not None else 0)
    return arr.slice(offset) if offset else arr


def case_mask(t_index, case):
    n, kind, ns, null_p, _validity, _voff, moff = case
    rng = np.random.default_rng([SEED, t_index, n, MASK_KINDS.index(kind)])
    if kind == "all_null":
        return mask_array(np.zeros(n, bool), ns, 0.0, moff, rng, all_null=True)
    return mask_array(selection(kind, n, rng), ns, null_p, moff, rng)


def take_tile(w, iw):
    """indices one warp covers per step of take_kernel: 32 lanes x V = 16 / max(index width, value width) x kUnroll"""
    return 32 * (16 // max(w, iw)) * UNROLL


def take_cases(t, it):
    """(indices, index offset, values null share, indices null share): k * tile +- 1 with k = 1 and k = kWarpsPerBlock + 1
    (a second CTA), one offset that breaks the indices' 16-byte alignment"""
    tile = take_tile(sr.byte_width(t), sr.byte_width(it))
    k = WARPS + 1
    return [(tile - 1, 0, 0.2, 0.0), (tile + 1, 0, 0.0, 0.2), (k * tile - 1, 1, 0.1, 0.1), (k * tile + 1, 0, 0.1, 0.1)]


def take_values_length(it):
    return min(np.iinfo(it.to_pandas_dtype()).max + 1, 3000)


BAND_KB = 1
BAND_VALUES = 40000
BAND_CASES = [(t, it) for t in (pa.int8(), pa.float16(), pa.binary(16)) for it in (pa.int32(), pa.uint32(), pa.int64(), pa.uint64())]
PARTITION_CASES = [(t, it) for t in (pa.binary(8), pa.timestamp("us")) for it in (pa.int32(), pa.uint64())]
BOOL_TILES = 65  # output tile t of the residue mask starts at bit t mod 64 of a word
TAKE_INDICES_LENGTHS = (1, 0xFFFF, 0x10000, 70001)
STRING_TAKE_COUNTS = (TAKE_TILE - 1, TAKE_TILE, TAKE_TILE + 1, 2 * TAKE_TILE + 1)
STRING_WIDE_ROWS = (20, 40)  # row lengths of the wide-tile cases: every full tile's output passes 32 KiB


# ---- the host's choices, restated --------------------------------------------------------------------------------------
def filter_regimes(n, sel, w, values_offset):
    """which template, compaction paths and look-back depth b2_filter uses for this input"""
    out = int(sel.sum())
    if out == 0:
        return {"empty"}
    vec_ok = values_offset * w % 16 == 0
    n_spans = -(-(-(-n // TILE)) // SPAN_TILES)
    reg = {"template:sparse" if out < n // 8 else "template:dense",
           "lookback:multi" if n_spans - 1 > LOOKBACK_STEP else "lookback:single"}
    r = 16 // w
    s = np.concatenate([sel, np.zeros(-n % CHUNK, bool)]).reshape(-1, CHUNK)
    counts = s.sum(axis=1)
    chunk = np.arange(len(counts))
    dense = vec_ok & (counts >= CHUNK // 8) & ((chunk + 1) * CHUNK <= n)
    if dense.any():
        reg.add("chunk:dense")
    rest = np.flatnonzero((counts > 0) & ~dense)
    groups = s[rest].reshape(len(rest), CHUNK // r, r).any(axis=2)
    start = rest[:, None] * CHUNK + np.arange(CHUNK // r)[None, :] * r
    vector = vec_ok & (start + r <= n)
    if (groups & vector).any():
        reg.add("chunk:vector")
    if (groups & ~vector).any():
        reg.add("chunk:scalar")
    return reg


def take_regimes(n, w, iw, index_offset):
    tile = take_tile(w, iw)
    vec_ok = index_offset * iw % 16 == 0
    reg = set()
    if vec_ok and n >= tile:
        reg.add("take:vector")
    if not vec_ok or n % tile:
        reg.add("take:scalar")
    return reg


def band_count(values_length, iw, band_kb):
    """take_bands with B2_TAKE_BAND_KB set, for values with nulls"""
    if iw not in (4, 8):
        return 1
    band = band_kb << 10
    k = -(-(values_length >> 3) // band)
    return k if 2 <= k <= 6 else 1


def bool_residue_selection(n, rng):
    """tile t keeps 1 + 64 j rows, so the survivors before tile t number t mod 64"""
    sel = np.zeros(n, bool)
    for tile in range(-(-n // TILE)):
        lo, m = tile * TILE, min(TILE, n - tile * TILE)
        sel[lo + rng.choice(m, min(m, 1 + 64 * (tile % 7)), replace=False)] = True
    return sel


def bool_residues(sel):
    tiles = -(-len(sel) // TILE)
    counts = np.array([sel[t * TILE:(t + 1) * TILE].sum() for t in range(tiles)])
    before = np.concatenate([[0], np.cumsum(counts)[:-1]])
    return set((before[counts > 0] % 64).tolist())


def coarse_shift(tile_bytes):
    """copy_tile_bytes: the smallest g >= 6 with tile_bytes >> g < 512"""
    g = 6
    while (tile_bytes >> g) >= 512:
        g += 1
    return g


def test_case_tables_reach_every_regime():
    required = {"template:sparse", "template:dense", "chunk:dense", "chunk:vector", "chunk:scalar", "lookback:multi",
                "lookback:single"}
    for ti, t in enumerate(FILTER_LAYOUTS):
        w = sr.byte_width(t)
        seen = set()
        for case in filter_cases(t):
            mask = case_mask(ti, case)
            seen |= filter_regimes(case[0], sr.selected(mask, case[2]), w, case[5])
        # a 16-byte row is one 16-byte load: with element-aligned values it never takes the scalar path
        want = required - ({"chunk:scalar"} if w == 16 else set())
        assert want <= seen, f"{t}: {sorted(want - seen)} not reached"
        kinds = {(c[2], c[4], c[5] * w % 16 == 0, c[6] % 8 == 0) for c in filter_cases(t)}
        assert {k[0] for k in kinds} == {sr.DROP, sr.EMIT_NULL} and {k[1] for k in kinds} == set(VALIDITY)
        assert {k[3] for k in kinds} == {True, False} and (w == 16 or {k[2] for k in kinds} == {True, False})
    for t in TAKE_LAYOUTS:
        for it in INDEX_TYPES:
            seen = set()
            for n, ioff, _, _ in take_cases(t, it):
                seen |= take_regimes(n, sr.byte_width(t), sr.byte_width(it), ioff)
            assert seen == {"take:vector", "take:scalar"}, (t, it, seen)
    assert {sr.byte_width(t) for t in TAKE_LAYOUTS} == {1, 2, 4, 8, 16}
    for t, it in BAND_CASES:
        assert band_count(BAND_VALUES, sr.byte_width(it), BAND_KB) >= 2, (t, it)
    assert {sr.byte_width(t) for t, _ in BAND_CASES} == {1, 2, 16}
    n = BOOL_TILES * TILE + 37
    assert bool_residues(bool_residue_selection(n, np.random.default_rng(SEED))) == set(range(64))
    assert {0xFFFF, 0x10000} <= set(TAKE_INDICES_LENGTHS)
    assert coarse_shift(TILE * STRING_WIDE_ROWS[0]) > 6 and coarse_shift(TAKE_TILE * STRING_WIDE_ROWS[0]) > 6
    assert {TAKE_TILE - 1, TAKE_TILE + 1} <= set(STRING_TAKE_COUNTS)


# ---- checks ------------------------------------------------------------------------------------------------------------
def check(got: DeviceArray, want: sr.Rows, msg=""):
    assert got.null_count == want.null_count(), f"{msg}: null_count {got.null_count} != {want.null_count()}"
    arr = got.to_arrow()
    arr.validate(full=True)
    sr.assert_rows_equal(arr, want, msg)
    return arr


def dev(arr, ctx):
    return DeviceArray.from_arrow(arr, ctx)


def values_view(ctx, base: DeviceArray, base_valid, t, n, offset, validity):
    """n rows of `base` from `offset`, without a bitmap, with it and its null count, or with it and null_count = -1"""
    data = base.buffers[1].ptr
    if validity == "none":
        return DeviceArray.from_pointers(ctx, t, n, data, offset=offset, keepalive=base)
    nc = -1 if validity == "unknown" else int((~base_valid[offset:offset + n]).sum())
    return DeviceArray.from_pointers(ctx, t, n, data, validity_ptr=base.buffers[0].ptr, null_count=nc, offset=offset,
                                     keepalive=base)


# ---- fixed-width Filter ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("ti", range(len(FILTER_LAYOUTS)), ids=[str(t) for t in FILTER_LAYOUTS])
def test_fixed_width_filter(ctx, ti):
    t = FILTER_LAYOUTS[ti]
    by_length = {}
    for case in filter_cases(t):
        by_length.setdefault(case[0], []).append(case)
    for n, cases in by_length.items():
        rng = np.random.default_rng([SEED, ti, n])
        m = n + max(VALUE_OFFSETS)
        raw = in_range_bytes(t, m, rng)
        valid = rng.random(m) >= 0.15
        valid[0] = False
        base = dev(pa.Array.from_buffers(t, m, [bitmap(valid), pa.py_buffer(raw.tobytes())], null_count=-1), ctx)
        identity_done = False
        for case in cases:
            _, kind, ns, _, validity, voff, _ = case
            dv = values_view(ctx, base, valid, t, n, voff, validity)
            ref = sr.Rows(t, "fixed", raw[voff:voff + n], valid[voff:voff + n] if validity != "none" else np.ones(n, bool))
            mask = case_mask(ti, case)
            dm = dev(mask, ctx)
            want = sr.filter(ref, mask, ns)
            msg = f"{t} n={n} {kind} {ns} {validity} voff={voff} moff={mask.offset}"
            check(bc.filter(dv, dm, ns), want, msg)
            assert bc.filter_output_size(dm, ns) == len(want), msg
            if kind == "random" and not identity_done and n > 1:  # Filter(v, m) == Take(v, take_indices_from_filter(m))
                identity_done = True
                idx = bc.take_indices_from_filter(dm, ns)
                check(bc.take(dv, idx), want, f"{msg} via take_indices")


@gpu
@pytest.mark.parametrize("n", TAKE_INDICES_LENGTHS)
def test_take_indices_from_filter(ctx, n):
    rng = np.random.default_rng([SEED, n])
    for ns in (sr.DROP, sr.EMIT_NULL):
        for null_p, moff in ((0.0, 0), (0.2, 5)):
            mask = mask_array(rng.random(n) < 0.4, ns, null_p, moff, rng)
            got = bc.take_indices_from_filter(dev(mask, ctx), ns)
            want = sr.take_indices(mask, ns)
            assert got.type == want.type == (pa.uint16() if n <= 0xFFFF else pa.uint32())
            check(got, want, f"n={n} {ns} {null_p}")


# ---- fixed-width Take --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("t", TAKE_LAYOUTS, ids=str)
def test_fixed_width_take(ctx, t):
    rng = np.random.default_rng([SEED, sr.byte_width(t), TAKE_LAYOUTS.index(t)])
    for it in INDEX_TYPES:
        vlen = take_values_length(it)
        for n, ioff, v_null, i_null in take_cases(t, it):
            values = fixed_array(t, vlen, rng, v_null, offset=3 if v_null else 0)
            idx = index_array(it, n, vlen, rng, i_null, ioff)
            dv, di = dev(values, ctx), dev(idx, ctx)
            check(bc.take(dv, di), sr.take(values, idx), f"{t} {it} n={n} ioff={ioff}")


def bad_index_case(it, tile):
    """(values length, indices, null rows, expected message): a bad index under a null at row 2, the first valid bad row at
    5 (negative for signed types; its low bits zero-extended would be in bounds), a second one in the scalar tail"""
    info = np.iinfo(it.to_pandas_dtype())
    w, signed = sr.byte_width(it), info.min < 0
    vlen = {1: 256 if signed else 200, 2: 40000}.get(w, 1000)
    if signed:
        first, later = {1: -100, 2: -30000, 4: -7, 8: -(1 << 40)}[w], -1
    else:
        first, later = (1 << 63) + 5 if w == 8 else int(info.max), int(info.max) - 1
    v = [i % 100 for i in range(tile + 1)]
    v[2], v[5], v[tile] = later, first, later
    return vlen, v, [2], f"Index {first} out of bounds"


@gpu
@pytest.mark.parametrize("t", TAKE_LAYOUTS, ids=str)
def test_fixed_width_take_index_errors(ctx, t):
    rng = np.random.default_rng(SEED)
    for it in INDEX_TYPES:
        vlen, v, nulls, message = bad_index_case(it, take_tile(sr.byte_width(t), sr.byte_width(it)))
        valid = np.ones(len(v), bool)
        valid[nulls] = False
        idx = pa.Array.from_buffers(it, len(v), [bitmap(valid), pa.py_buffer(np.array(v, it.to_pandas_dtype()).tobytes())],
                                    null_count=len(nulls))
        values = fixed_array(t, vlen, rng, 0.1)
        with pytest.raises(pa.ArrowIndexError) as want:
            sr.take(values, idx)
        assert str(want.value) == message
        dv, di = dev(values, ctx), dev(idx, ctx)
        for boundscheck in (True, False):
            with pytest.raises(pa.ArrowIndexError) as got:
                bc.take(dv, di, boundscheck=boundscheck)
            assert str(got.value) == message, (t, it, boundscheck)
        # the same indices with every bad row null: the one under the null at row 2 is never read
        valid[[5, len(v) - 1]] = False
        idx = pa.Array.from_buffers(it, len(v), [bitmap(valid), idx.buffers()[1]], null_count=3)
        check(bc.take(dv, dev(idx, ctx)), sr.take(values, idx), f"{t} {it} bad rows under nulls")


@gpu
@pytest.mark.parametrize("t,it", BAND_CASES, ids=str)
def test_take_validity_bands(ctx, monkeypatch, t, it):
    """B2_TAKE_BAND_KB cuts the values' bitmap into bands: the gather probes band 0, one follow-up launch per band clears
    the rest"""
    monkeypatch.setenv("B2_TAKE_BAND_KB", str(BAND_KB))
    rng = np.random.default_rng([SEED, sr.byte_width(t), sr.byte_width(it)])
    values = fixed_array(t, BAND_VALUES, rng, 0.3)
    tile = take_tile(sr.byte_width(t), sr.byte_width(it))
    for n, ioff, i_null in ((3 * tile + 5, 0, 0.0), (WARPS * tile + 1, 1, 0.1)):
        idx = index_array(it, n, BAND_VALUES, rng, i_null, ioff)
        check(bc.take(dev(values, ctx), dev(idx, ctx)), sr.take(values, idx), f"{t} {it} n={n}")


@gpu
@pytest.mark.parametrize("t,it", PARTITION_CASES, ids=str)
def test_take_partitioned_layouts(ctx, monkeypatch, t, it):
    monkeypatch.setenv("B2_TAKE_PARTITION", "1")
    rng = np.random.default_rng(SEED + 7)
    values = fixed_array(t, 3000, rng, 0.2)
    idx = index_array(it, 5000, 3000, rng, 0.1, 1)
    check(bc.take(dev(values, ctx), dev(idx, ctx)), sr.take(values, idx), f"{t} {it}")


@gpu
@pytest.mark.parametrize("t", [pa.binary(3), pa.binary(12), pa.binary(17)], ids=str)
def test_unsupported_fixed_size_binary_widths_are_refused(ctx, t):
    """the kernels move rows of 1, 2, 4, 8 or 16 bytes; other widths are refused, not computed (the reference takes any)"""
    values = dev(fixed_array(t, 10, np.random.default_rng(SEED), 0.0), ctx)
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.filter(values, dev(pa.array([True, False] * 5), ctx))
    with pytest.raises(pa.ArrowNotImplementedError):
        bc.take(values, dev(pa.array([0, 9], pa.int32()), ctx))


# ---- bool --------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("ns", [sr.DROP, sr.EMIT_NULL])
def test_bool_filter_every_word_residue(ctx, ns):
    n = BOOL_TILES * TILE + 37  # the last tile and most output tiles end inside a word
    rng = np.random.default_rng(SEED + 11)
    sel = bool_residue_selection(n, rng)
    assert bool_residues(sel) == set(range(64))
    for voff, moff, v_null, m_null in ((0, 0, 0.0, 0.0), (5, 3, 0.2, 0.1), (64, 13, 0.1, 0.3)):
        values = bool_array(n, rng, 0.5, v_null, voff)
        mask = mask_array(sel, ns, m_null, moff, rng)
        check(bc.filter(dev(values, ctx), dev(mask, ctx), ns), sr.filter(values, mask, ns), f"{voff} {moff} {v_null}")
        if m_null == 0:  # the dense other half too
            mask = mask_array(~sel, ns, 0.0, moff, rng)
            check(bc.filter(dev(values, ctx), dev(mask, ctx), ns), sr.filter(values, mask, ns), "complement")


@gpu
def test_bool_take(ctx):
    rng = np.random.default_rng(SEED + 12)
    for vlen, v_null in ((100, 0.3), (5000, 0.0), (5000, 0.2)):
        values = bool_array(vlen, rng, 0.5, v_null, 3)
        for it in INDEX_TYPES:
            for n, i_null, ioff in ((31, 0.0, 0), (4097, 0.2, 1), (40001, 0.1, 0)):
                idx = index_array(it, n, min(vlen, 128) if sr.byte_width(it) == 1 else vlen, rng, i_null, ioff)
                check(bc.take(dev(values, ctx), dev(idx, ctx)), sr.take(values, idx), f"{vlen} {it} n={n}")
    values = bool_array(200, rng, 0.5, 0.1)
    for it in INDEX_TYPES:
        _, v, nulls, _ = bad_index_case(it, 64)  # every bad value is out of bounds for 200 values too
        valid = np.ones(len(v), bool)
        valid[nulls] = False
        idx = pa.Array.from_buffers(it, len(v), [bitmap(valid), pa.py_buffer(np.array(v, it.to_pandas_dtype()).tobytes())],
                                    null_count=len(nulls))
        with pytest.raises(pa.ArrowIndexError) as got:
            bc.take(dev(values, ctx), dev(idx, ctx))
        with pytest.raises(pa.ArrowIndexError) as want:
            sr.take(values, idx)
        assert str(got.value) == str(want.value)


# ---- utf8 / binary -----------------------------------------------------------------------------------------------------
def strings_from(t, rows, valid=None, offset=0):
    """an array of type t holding `rows` (bytes), sliced at `offset`"""
    lens = np.array([len(r) for r in rows], np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64 if sr.offset_width(t) == 8 else np.int32)
    bufs = [None if valid is None else bitmap(valid), pa.py_buffer(offs.tobytes()), pa.py_buffer(b"".join(rows))]
    arr = pa.Array.from_buffers(t, len(rows), bufs, null_count=-1 if valid is not None else 0)
    return arr.slice(offset) if offset else arr


def empty_run_rows(n, rng):
    """rows of 16 bytes and of 1-17 bytes separated by runs of empty strings, so outputs put empty rows at 16-byte
    boundaries and chunks start mid-row"""
    rows = []
    while len(rows) < n:
        rows.append(bytes(rng.integers(97, 123, int(rng.choice([16, 16, 32, 1, 7, 15, 17])), dtype=np.uint8)))
        rows.extend([b""] * int(rng.integers(0, 5)))
    return rows[:n]


def shifted(ctx, arr: pa.Array, shift: int) -> DeviceArray:
    """arr on the device with its data buffer starting `shift` bytes past an 8-byte boundary"""
    base = dev(arr, ctx)
    data = np.frombuffer(arr.buffers()[2], np.uint8)
    raw = ctx.alloc(len(data) + 32)
    host = np.ascontiguousarray(data)
    ctx.h2d(raw.ptr + shift, host.ctypes.data, len(host))
    ctx.sync()
    return DeviceArray.from_pointers(ctx, arr.type, len(arr), base.buffers[1].ptr,
                                     validity_ptr=base.buffers[0].ptr if base.buffers[0] is not None else 0,
                                     null_count=arr.null_count, offset=arr.offset, data2_ptr=raw.ptr + shift,
                                     keepalive=(base, raw))


@gpu
@pytest.mark.parametrize("t", STRING_TYPES, ids=str)
def test_string_filter_take_edges(ctx, t):
    rng = np.random.default_rng(SEED + 13)
    n = 3 * TILE + 5
    wide = random_array(t, n, 0.1, SEED + 1, lo=STRING_WIDE_ROWS[0], hi=STRING_WIDE_ROWS[1], offset=3)
    runs = strings_from(t, empty_run_rows(n + 2, rng), rng.random(n + 2) >= 0.1, offset=2)
    runs_nonnull = strings_from(t, empty_run_rows(n, rng))
    for values in (wide, runs, runs_nonnull):
        for shift in (0, 3, 5):
            dv = dev(values, ctx) if shift == 0 else shifted(ctx, values, shift)
            for ns in (sr.DROP, sr.EMIT_NULL):
                for p_true, m_null in ((1.0, 0.0), (0.6, 0.2), (0.05, 0.1)):
                    mask = mask_array(rng.random(n) < p_true, ns, m_null, 1, rng)
                    check(bc.filter(dv, dev(mask, ctx), ns), sr.filter(values, mask, ns), f"{t} shift={shift} {ns} {p_true}")
            for count in STRING_TAKE_COUNTS:
                for it, i_null, ioff in ((pa.int32(), 0.0, 0), (pa.uint64(), 0.1, 3), (pa.int16(), 0.05, 1)):
                    idx = index_array(it, count, n, rng, i_null, ioff)
                    check(bc.take(dv, dev(idx, ctx)), sr.take(values, idx), f"{t} shift={shift} take {count} {it}")
    # the first bad row is reported
    idx = pa.array([0, None, n + 4, -3, n], pa.int64())
    with pytest.raises(pa.ArrowIndexError, match=f"^Index {n + 4} out of bounds$"):
        bc.take(dev(wide, ctx), dev(idx, ctx))


@gpu
@pytest.mark.parametrize("it", INDEX_TYPES, ids=str)
def test_dictionary_filter_take(ctx, it):
    rng = np.random.default_rng(SEED + 14)
    d = dictionary_array(it, 9000, rng)
    dd = dev(d, ctx)
    for ns in (sr.DROP, sr.EMIT_NULL):
        mask = mask_array(rng.random(9000) < 0.3, ns, 0.1, 3, rng)
        check(bc.filter(dd, dev(mask, ctx), ns), sr.filter(d, mask, ns), f"{it} {ns}")
    for jt in (pa.int8(), pa.uint32(), pa.int64()):
        idx = index_array(jt, 3001, 9000, rng, 0.1, 1)
        check(bc.take(dd, dev(idx, ctx)), sr.take(d, idx), f"{it} {jt}")


# ---- int32-offset capacity (about 5 GiB of device memory) ---------------------------------------------------------------
BIG_BYTES = 5 << 30
MIB = 1 << 20


@pytest.fixture()
def big_memory(ctx):
    import torch
    gc.collect()
    torch.cuda.empty_cache()  # hand cached blocks back so the context's own pool can allocate them
    ctx.sync()
    ctx.trim()
    free, _ = torch.cuda.mem_get_info()
    if free < BIG_BYTES:
        pytest.skip(f"needs ~{BIG_BYTES >> 30} GiB of free device memory")
    print(f"[free device memory: {free / 2**30:.1f} GiB]")
    yield torch
    gc.collect()
    torch.cuda.empty_cache()
    ctx.sync()
    ctx.trim()


def device_bytes(torch, ptr, nbytes):
    """zero-copy torch view of nbytes of device memory"""
    class _Cai:
        pass
    shim = _Cai()
    shim.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2,
                                     "strides": (1,)}
    return torch.as_tensor(shim, device="cuda")


@gpu
def test_capacity_take_int32_offsets(ctx, big_memory):
    """2047 rows of 1 MiB and one more: 2^31 - 2 output bytes fit int32 offsets, 2^31 - 1 do not (kOffsetLimit), a null
    last row adds nothing, and 64-bit offsets hold all of them"""
    torch = big_memory
    sizes = [MIB, MIB - 2, MIB - 1]
    chars = np.random.default_rng(SEED).integers(0, 256, sum(sizes), dtype=np.uint8)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    starts = offs[:-1].tolist()
    for t in (pa.binary(), pa.large_binary()):
        values = pa.Array.from_buffers(t, 3, [None, pa.py_buffer(offs.astype(np.int64 if sr.offset_width(t) == 8 else np.int32).tobytes()),
                                              pa.py_buffer(chars.tobytes())])
        dv = dev(values, ctx)
        rows_t = [torch.from_numpy(chars[s:s + z].copy()).cuda() for s, z in zip(starts, sizes)]
        for last, last_null in ((1, False), (2, False), (2, True)):
            idx = pa.array([0] * 2047 + [None if last_null else last], pa.int32())
            taken = [sizes[0]] * 2047 + ([] if last_null else [sizes[last]])
            if sr.offset_width(t) == 4 and sr.take_overflows(taken):
                with pytest.raises(pa.ArrowInvalid, match=f"^{sr.TAKE_CAPACITY_MESSAGE}$"):
                    bc.take(dv, dev(idx, ctx))
                continue
            out = bc.take(dv, dev(idx, ctx))
            ctx.sync()
            assert len(out) == 2048 and out.null_count == int(last_null)
            got_offs = out.buffers[1].to_numpy(sr.offset_width(t) * 2049).view(np.int64 if sr.offset_width(t) == 8 else np.int32)
            want_offs = np.concatenate([[0], np.cumsum(taken + [0] * last_null)])
            assert np.array_equal(got_offs.astype(np.int64), want_offs), (t, last, last_null)
            total = int(want_offs[-1])
            assert total == (1 << 31) - 2 - (MIB - 2) * last_null + (last == 2 and not last_null)
            data = device_bytes(torch, out.buffers[2].ptr, total)
            for r in range(0, 2047, 256):
                k = min(256, 2047 - r)
                assert torch.equal(data[r * MIB:(r + k) * MIB].view(k, MIB), rows_t[0].expand(k, MIB)), (t, r)
            if not last_null:
                assert torch.equal(data[2047 * MIB:], rows_t[last])
            del out, data
        del dv


@gpu
def test_capacity_filter_keeps_2gib_minus_one(ctx, big_memory):
    """a utf8 / binary array with int32 offsets holds at most 2^31 - 1 value bytes, and Filter keeps all of them: its
    output is never larger than its input, so it has no capacity error (the reference has none either)"""
    torch = big_memory
    total = (1 << 31) - 1
    n, size = 1 << 15, 1 << 16  # 32768 rows of 64 KiB, the last one byte shorter: 8 tiles
    gen = torch.Generator(device="cuda").manual_seed(SEED)
    offs = (torch.arange(n + 1, dtype=torch.int64, device="cuda") * size).clamp_(max=total).to(torch.int32)
    data = torch.empty(total + 64, dtype=torch.uint8, device="cuda")
    data.random_(0, 256, generator=gen)
    torch.cuda.synchronize()
    values = DeviceArray.from_pointers(ctx, pa.binary(), n, offs.data_ptr(), data2_ptr=data.data_ptr(), keepalive=(offs, data))
    out = bc.filter(values, dev(pa.array(np.ones(n, bool)), ctx))
    ctx.sync()
    assert len(out) == n and out.null_count == 0
    got_offs = torch.from_numpy(out.buffers[1].to_numpy(4 * (n + 1)).view(np.int32).copy()).cuda()
    assert torch.equal(got_offs, offs)
    assert torch.equal(device_bytes(torch, out.buffers[2].ptr, total), data[:total])
